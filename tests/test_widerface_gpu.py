"""A live Net that changes its input size between forwards, and the WIDER FACE driver loop built on it.

(a) One net goes through a sequence of input shapes (shrink, grow, back to an earlier one).  At every step its outputs,
    proposals_score, the cascade stage blobs the drivers read and the final detections equal, bit for bit, those of a
    net built afresh at that shape with the same weights; a shape change re-packs no weights.  Eager and CUDA-graph
    forwards, fp32-faithful and plain bf16, models.widerface and models.widerface_cascade.
(b) widerface.run (size-bucketed batches) against the drivers' loop (one frame per forward, each at its own net size):
    every image's detections are bit-identical, and (c) so are the result files written from both.
The convolution launch-plan cache stays bounded: revisiting shapes adds no plans."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(2, 128, 192), (1, 96, 160), (3, 160, 224), (2, 128, 192)]
STAGES = ["proposals", "proposals_2nd", "proposals_3rd", "output_bbox_1st", "output_bbox_2nd", "output_bbox_3rd",
          "cls_prob_1st", "cls_prob_2nd", "cls_prob_3rd", "cls_prob_3rd_avg"]


@pytest.fixture()
def side_stream(cuda):
    from mscnn_b200 import net as mnet
    s = torch.cuda.Stream()
    prev = torch.cuda.current_stream()
    torch.cuda.set_stream(s)
    mnet.set_stream(s.cuda_stream)
    yield s
    torch.cuda.synchronize()
    torch.cuda.set_stream(prev)
    mnet.set_stream(prev.cuda_stream)


def _proto(kind, n, h, w):
    from mscnn_b200 import models
    return getattr(models, kind)(h, w, batch=n)


def _results(net, kind, n, h, w):
    """Everything the drivers read from one forward, as host arrays."""
    from mscnn_b200 import net as mnet
    res = {k: net.blob(k) for k in net.outputs}
    res["proposals_score"] = net.blob("proposals_score")
    if kind == "widerface_cascade":
        res.update({k: net.blob(k) for k in STAGES})
    res["num_proposals"] = np.array([net.num_proposals(i) for i in range(n)])
    cfg, classes = mnet.widerface_detect_cfg(h, w)
    dets = torch.zeros((n, 1, cfg.max_rois_per_image, 5), device="cuda")
    cnt = torch.zeros((n, 1), dtype=torch.int32, device="cuda")
    if kind == "widerface_cascade":
        net.detect_cascade_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr(), stage="3rd",
                                   cls_prob="cls_prob_3rd_avg")
    else:
        net.detect_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    res["dets"], res["counts"] = dets.cpu().numpy(), cnt.cpu().numpy()
    return res


def _assert_same(got, want, step):
    assert sorted(got) == sorted(want), step
    for k in want:
        a, b = np.ascontiguousarray(got[k]), np.ascontiguousarray(want[k])
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), (step, k)


CASES = [("widerface", "fp32", False), ("widerface", "bf16", False), ("widerface_cascade", "fp32", False),
         ("widerface_cascade", "bf16", False), ("widerface", "fp32", True), ("widerface_cascade", "fp32", True)]


@pytest.mark.parametrize("kind,precision,graph", CASES)
def test_live_net_through_shapes_equals_fresh_nets(request, cuda, kind, precision, graph):
    from mscnn_b200 import capi, net as mnet, synth
    if graph:
        request.getfixturevalue("side_stream")          # a graph cannot be captured on the legacy default stream
    L = capi.lib()
    try:
        mnet.set_precision(precision)
        weights = None
        want = []
        # the fresh nets first: none of them runs while the live net holds a captured graph
        for step, (n, h, w) in enumerate(SHAPES):
            fresh = mnet.Net(_proto(kind, n, h, w))
            weights = weights or synth.make_weights(fresh.layers())
            fresh.set_params(weights)
            fresh.forward(data=synth.make_images(n, h, w, first_index=10 * step))
            want.append(_results(fresh, kind, n, h, w))
            assert int(want[-1]["counts"].sum()) > 0
            del fresh
        n0, h0, w0 = SHAPES[0]
        live = mnet.Net(_proto(kind, n0, h0, w0))
        live.set_params(weights)
        live.set_graph(graph)
        replays = 0
        for step, (n, h, w) in enumerate(SHAPES):
            live.reshape_input("data", n, 3, h, w)
            images = synth.make_images(n, h, w, first_index=10 * step)
            launches = []
            for _ in range(3 if graph else 2):   # graph: eager after the shape change, then capture, then replay
                live.set_input("data", images)
                torch.cuda.synchronize()
                c0 = L.mscnn_kernel_launch_count()
                live.forward_only()
                torch.cuda.synchronize()
                launches.append(L.mscnn_kernel_launch_count() - c0)
                replays += int(live.graph_replayed())
                _assert_same(_results(live, kind, n, h, w), want[step], (step, (n, h, w), len(launches)))
            if not graph and step > 0:   # the first forward at a new shape packs no weights: it launches what the
                assert launches[0] == launches[1], (step, launches)          # next one does
        if graph:
            assert replays >= len(SHAPES), replays
    finally:
        mnet.set_precision("fp32")


def test_conv_plan_cache_stays_bounded(cuda):
    """Plans are keyed by descriptor (tensor addresses and extents).  Largest shape first, as plan_batches orders the
    groups, so that the buffers stop moving: a second pass over the same shapes then finds every plan it needs."""
    from mscnn_b200 import capi, net as mnet, synth
    L = capi.lib()
    mnet.set_precision("fp32")
    sizes = [(224, 288), (192, 256), (160, 256), (160, 224), (128, 192), (96, 160), (96, 128), (64, 96)]
    net = mnet.Net(_proto("widerface", 1, *sizes[0]))       # creating a net empties the plan cache
    net.set_params(synth.make_weights(net.layers()))
    counts = []
    for p in range(2):
        for i, (h, w) in enumerate(sizes):
            net.reshape_input("data", 1, 3, h, w)
            net.set_input("data", synth.make_images(1, h, w, first_index=i))
            net.forward_only()
            net.num_proposals()
            counts.append(L.mscnn_conv_plan_count())
    first, second = counts[:len(sizes)], counts[len(sizes):]
    assert all(b > a for a, b in zip(first, first[1:])), first      # each new shape adds its convolutions' plans
    assert second == [first[-1]] * len(sizes), (first, second)      # revisited shapes add none
    assert first[-1] <= 4096


# --------------------------------------------------------------------------------------------- the driver loop
ORG = [(120, 150), (100, 150), (130, 170), (150, 200), (90, 130)]


def _frames():
    rng = np.random.default_rng(2024)
    out = []
    for k in range(10):
        h, w = ORG[k % len(ORG)]
        im = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        im[: h // 4, : w // 4] = 255
        out.append(im)
    return out


def _driver_loop(net, frames, names, cascade):
    """run_mscnn_detection.m:68-146: one frame per forward at its own net size, the ratios in the cfg."""
    from mscnn_b200 import net as mnet, ops
    out = {}
    for name, im in zip(names, frames):
        oh, ow = im.shape[:2]
        rz = ops.widerface_net_size(oh, ow, 0, 0, 3072)
        net.reshape_input("data", 1, 3, *rz)
        pre = ops.Preprocess((oh, ow), rz)       # kept until the synchronize below: its kernels are in flight
        net.set_input_images("data", pre, im[None])
        net.forward_only()
        cfg, classes = mnet.widerface_detect_cfg(*rz, org_hw=(oh, ow))
        dets = torch.zeros((1, 1, cfg.max_rois_per_image, 5), device="cuda")
        cnt = torch.zeros((1, 1), dtype=torch.int32, device="cuda")
        if cascade:
            net.detect_cascade_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr(), stage="3rd",
                                       cls_prob="cls_prob_3rd_avg")
        else:
            net.detect_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr())
        torch.cuda.synchronize()
        out[name] = dets[0, 0, :int(cnt[0, 0])].cpu().numpy()
    return out


@pytest.mark.parametrize("kind", ["widerface", "widerface_cascade"])
def test_run_equals_the_driver_loop_and_writes_the_same_files(cuda, tmp_path, kind):
    from mscnn_b200 import net as mnet, synth, widerface
    from oracle import port
    mnet.set_precision("fp32")
    frames = _frames()
    names = [f"9_Press_Conference_Press_Conference_9_{k}" for k in range(len(frames))]
    net_sizes = {port.widerface_net_size(h, w, 0, 0, 3072) for h, w in ORG}
    assert len(net_sizes) >= 3
    budget = 3 * 128 * 160                       # the 128 x 160 group (4 frames) runs as two batches
    plan = widerface.plan_batches([f.shape[:2] for f in frames], pixel_budget=budget)
    assert len(plan) > len(net_sizes) and max(len(idx) for _, idx in plan) > 1
    cascade = kind == "widerface_cascade"
    loop_net = mnet.Net(_proto(kind, 1, 96, 128))
    weights = synth.make_weights(loop_net.layers())
    loop_net.set_params(weights)
    want = _driver_loop(loop_net, frames, names, cascade)
    net = mnet.Net(_proto(kind, 1, 96, 128))
    net.set_params(weights)
    got = widerface.run(net, frames, names, cascade=cascade, pixel_budget=budget)
    assert list(got) == names
    assert sum(len(v) for v in want.values()) > 0
    for k in names:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
        oh, ow = frames[names.index(k)].shape[:2]
        if len(got[k]):   # original-image coordinates, clipped to the image (the cascade's w = x2 - x1 + 1 may reach
            right = ow + (1 if cascade else 0) # one pixel past it, run_cascademscnn.m:109-111)
            assert np.all(got[k][:, :2] >= 0) and np.all(got[k][:, 0] + got[k][:, 2] <= right * (1 + 1e-6))
    # the same net again, default batching: the preprocessing plans come from the cache passed in
    plans = {}
    again = widerface.run(net, frames, names, cascade=cascade, plans=plans)
    assert sorted(plans) == sorted(net_sizes)
    for k in names:
        assert again[k].tobytes() == want[k].tobytes(), k
    # (c) the result files of both runs, byte for byte
    widerface.write_results(tmp_path / "loop" / "9--Press_Conference", want)
    widerface.write_results(tmp_path / "run" / "9--Press_Conference", got)
    for k in names:
        a = (tmp_path / "loop" / "9--Press_Conference" / f"{k}.txt").read_bytes()
        b = (tmp_path / "run" / "9--Press_Conference" / f"{k}.txt").read_bytes()
        assert a == b and a.startswith(f"{k}\n{len(want[k])}\n".encode()), k
