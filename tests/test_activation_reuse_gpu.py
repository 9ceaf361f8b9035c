"""Activation reuse (Net.set_activation_reuse) on the GPU.

(a) A net that reuses activation memory computes, bit for bit, what the same net without reuse computes: the net
    outputs, the blobs the post-process reads and the final detections, fp32-faithful and bf16, eager and CUDA-graph
    replayed, for the 8s golden net, mscnn-7s-576-2x (Deconvolution) and both cascade nets.  Every forward launches as
    many kernels as without reuse, and no planned blob is ever found off its arena slot.
(b) The WIDER 12s net through a sequence of net sizes (it re-plans at each new size) equals the run without reuse, in
    both precisions, eager and with graph mode on.
(b2) After a full forward, a partial forward from a later layer, with the blobs it reads from before its start kept,
    runs and equals the same sequence without reuse.
(c) The device memory a reusing net takes over its first forward stays within its arena plus the blobs outside it
    (plus a stated slack for weights, packed images and workspaces), and well below the same net without reuse.
(d) A released blob raises in Python with the message, and mscnn_net_get_blob returns MSCNN_ERR_INVALID.
(e) drivers.run (one plain and one cascade spec) and widerface.run over two sharing nets that reuse, in two threads,
    equal the one-net run without reuse."""
import re

import numpy as np
import pytest
import torch

from test_drivers_gpu import GOLD, NET_HW, ORG, _deploy, _frame

pytestmark = pytest.mark.gpu

NETS = {"kitti_8s": ("kitti_car/mscnn-8s-768-trainval", (192, 640), "kitti_car"),
        "kitti_7s_2x": ("kitti_car/mscnn-7s-576-2x", (192, 640), "kitti_car"),
        "kitti_cascade": ("kitti_car/cascade-mscnn-7s-576-2x-trainval", (192, 640), "kitti_car_cascade"),
        "citypersons_cascade": ("citypersons/cascade-mscnn-8s-1344-2x", (336, 672), "citypersons")}


def _proto(rel, n, h, w):
    import tarfile
    with tarfile.open(GOLD / "deploy.tar.xz") as t:
        text = t.extractfile(f"deploy/{rel}/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: \d+\s+input_dim: \d+",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def _launches():
    from mscnn_b200 import capi
    return int(capi.lib().mscnn_kernel_launch_count())


def _run(net, spec, images, net_hw):
    """Outputs, the post-process blobs and the final detections of one forward, and its kernel launches."""
    from mscnn_b200 import net as mnet
    torch.cuda.synchronize()
    k0 = _launches()
    out = net.forward(data=images)
    torch.cuda.synchronize()
    launches = _launches() - k0
    for b in spec.blobs:
        out[b] = net.blob(b)
    out["num_proposals"] = np.array([net.num_proposals()])
    cfg, classes = spec.detect_cfg(net_hw)
    n = images.shape[0]
    with torch.cuda.stream(mnet._net_stream()):
        dets = torch.zeros((n, len(spec.cls_ids), cfg.max_rois_per_image, 5), device="cuda")
        cnt = torch.zeros((n, len(spec.cls_ids)), dtype=torch.int32, device="cuda")
        if spec.cascade:
            net.detect_cascade_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr(), cls_prob=spec.blobs[1])
        else:
            net.detect_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr())
        out["dets"], out["counts"] = dets.cpu().numpy(), cnt.cpu().numpy()
    return out, launches


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


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", sorted(NETS))
def test_reuse_equals_no_reuse(request, cuda, name, precision, graph):
    from mscnn_b200 import drivers, net as mnet, synth
    if graph:
        request.getfixturevalue("side_stream")
    rel, (h, w), spec_name = NETS[name]
    spec = drivers.SPECS[spec_name]
    mnet.set_precision(precision)
    try:
        proto = _proto(rel, 2, h, w)
        batches = [synth.make_images(2, h, w, first_index=2 * s) for s in range(3)]
        off = mnet.Net(proto)
        weights = synth.make_weights(off.layers())
        off.set_params(weights)
        off.set_graph(graph)
        on = mnet.Net(proto)
        on.share_trained_layers_with(off)
        on.set_activation_reuse(True, spec.blobs)
        on.set_graph(graph)
        _run(off, spec, batches[0], (h, w))    # packs the weights both nets read, outside the launch counts below
        replays = 0
        for rnd in range(2):
            for k, x in enumerate(batches):
                want, n_off = _run(off, spec, x, (h, w))
                got, n_on = _run(on, spec, x, (h, w))
                replays += int(on.graph_replayed())
                assert n_on == n_off, (rnd, k)
                assert sorted(got) == sorted(want)
                for key in want:
                    assert got[key].shape == want[key].shape and got[key].tobytes() == want[key].tobytes(), (rnd, k, key)
        assert want["counts"].sum() > 0
        if graph:
            assert replays >= 4, replays
        arena, without = on.activation_bytes()
        assert 0 < arena < without
        assert on.activation_misses() == 0
    finally:
        mnet.set_precision("fp32")


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_widerface_through_sizes_equals_no_reuse(request, cuda, precision, graph):
    from mscnn_b200 import models, net as mnet, synth, widerface
    if graph:
        request.getfixturevalue("side_stream")
    mnet.set_precision(precision)
    try:
        _widerface_through_sizes(graph)
    finally:
        mnet.set_precision("fp32")


def _widerface_through_sizes(graph):
    from mscnn_b200 import models, net as mnet, synth, widerface
    rng = np.random.default_rng(77)
    sizes = [(120, 150), (100, 150), (130, 170), (150, 200), (90, 130), (200, 120)]
    frames = []
    for k in range(12):
        h, w = sizes[k % len(sizes)]
        im = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        im[: h // 4, : w // 4] = 255
        frames.append(im)
    names = [f"img_{k}" for k in range(len(frames))]
    proto = models.widerface(96, 128, batch=1)
    off = mnet.Net(proto)
    weights = synth.make_weights(off.layers())
    off.set_params(weights)
    on = mnet.Net(proto)
    on.share_trained_layers_with(off)
    on.set_activation_reuse(True)
    for net in (off, on):
        net.set_graph(graph)
    budget = 3 * 128 * 160
    want = widerface.run(off, frames, names, pixel_budget=budget)
    assert sum(len(v) for v in want.values()) > 0
    for _ in range(2):                             # every size again: plans made before are re-made, the arena kept
        got = widerface.run(on, frames, names, pixel_budget=budget)
        for k in names:
            assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
    assert set(on.reuse_keep) == {"proposals_score", "cls_pred", "bbox_pred"}
    assert on.activation_misses() == 0


def test_partial_forward_after_a_full_one(cuda):
    from mscnn_b200 import drivers, net as mnet, synth
    mnet.set_precision("fp32")
    spec = drivers.KITTI_CAR
    proto = _proto("kitti_car/mscnn-8s-768-trainval", 2, 192, 640)
    off = mnet.Net(proto)
    off.set_params(synth.make_weights(off.layers()))
    on = mnet.Net(proto)
    on.share_trained_layers_with(off)
    start = "conv5_1"
    s = on.layer_names.index(start)
    on.set_activation_reuse(True)
    plan = [line.split() for line in on.activation_plan().splitlines()]
    # the planned storages written before `start` and read at or after it
    needed = [b for b, _, span, where in plan if where.startswith("@") and int(span.split("-")[0]) < s <= int(span.split("-")[1])]
    assert needed
    on.set_activation_reuse(True, list(needed) + list(spec.blobs))
    for k in range(2):
        x = synth.make_images(2, 192, 640, first_index=2 * k)
        want, got = {}, {}
        for net, res in ((off, want), (on, got)):
            net.forward(data=x)
            net.forward_only(start=start)
            for b in net.outputs + list(spec.blobs) + needed:
                res[b] = net.blob(b)
            res["num_proposals"] = np.array([net.num_proposals()])
        for key in want:
            assert got[key].shape == want[key].shape and got[key].tobytes() == want[key].tobytes(), (k, key)
    assert on.activation_misses() == 0


def _outside_bytes(net):
    return sum(int(line.split()[1]) for line in net.activation_plan().splitlines() if not line.split()[3].startswith("@"))


def test_memory_of_a_reusing_net(cuda):
    from mscnn_b200 import net as mnet, synth
    mnet.set_precision("fp32")
    n, h, w = 2, 384, 1280
    proto = _proto("kitti_car/mscnn-8s-768-trainval", n, h, w)
    images = synth.make_images(n, h, w)
    owner = mnet.Net(proto)
    weights = synth.make_weights(owner.layers())
    owner.set_params(weights)
    owner.forward(data=images)                   # weights uploaded and packed: the nets below add activations only
    torch.cuda.synchronize()

    def first_forward(reuse):
        free0 = torch.cuda.mem_get_info()[0]
        net = mnet.Net(proto)
        net.share_trained_layers_with(owner)
        if reuse:
            net.set_activation_reuse(True)
        net.forward(data=images)
        torch.cuda.synchronize()
        return net, free0 - torch.cuda.mem_get_info()[0]

    on, grow_on = first_forward(True)
    arena, without = on.activation_bytes()
    outside = _outside_bytes(on)
    # slack: per-layer bias pads, BoxOutput's workspace, the thread's scratch, pinned staging and allocation rounding
    slack = 256 << 20
    assert grow_on <= arena + outside + slack, (grow_on, arena, outside)
    del on
    torch.cuda.synchronize()
    off, grow_off = first_forward(False)
    assert grow_on < 0.6 * grow_off, (grow_on, grow_off)
    assert grow_off >= without                    # without reuse every planned storage has memory of its own


def test_released_blob_raises(cuda):
    from mscnn_b200 import capi, net as mnet, synth
    mnet.set_precision("fp32")
    proto = _proto("kitti_car/mscnn-8s-768-trainval", 1, 192, 640)
    net = mnet.Net(proto)
    net.set_params(synth.make_weights(net.layers()))
    net.set_activation_reuse(True, ["conv4_3"])
    out = net.forward(data=synth.make_images(1, 192, 640))
    assert set(out) == set(net.outputs)
    net.blob("conv4_3")                           # kept: readable
    assert net.blob_shape("conv1_1") == (1, 64, 192, 640)                  # a released blob keeps its shape
    with pytest.raises(capi.MscnnError, match="blob 'conv1_1' was released by activation reuse: its storage is reused "
                                              "after layer 'conv1_2' .*keep it readable by naming 'conv1_1'"):
        net.blob("conv1_1")
    buf = np.empty(64 * 192 * 640, dtype=np.float32)
    assert net._L.mscnn_net_get_blob(net._h, b"conv1_1", buf.ctypes.data, buf.size) == capi.ERR_INVALID
    # keeping it makes it readable after the next forward
    net.set_activation_reuse(True, ["conv4_3", "conv1_1"])
    net.forward(data=synth.make_images(1, 192, 640))
    assert net.blob("conv1_1").shape == (1, 64, 192, 640)
    # fc6 is planned planes only and not reused after its last reader: readable, and the NCHW buffer that host read
    # made is the host's, not a miss of the next forward
    assert "fc6" in [line.split()[0] for line in net.activation_plan().splitlines() if line.split()[3].startswith("@")]
    net.blob("fc6")
    net.forward(data=synth.make_images(1, 192, 640))
    assert net.activation_misses() == 0


@pytest.mark.parametrize("name", ["kitti_car", "citypersons"])
def test_driver_run_over_two_reusing_nets(cuda, name):
    from mscnn_b200 import drivers, net as mnet, synth
    mnet.set_precision("fp32")
    spec = drivers.SPECS[name]
    net_hw = NET_HW[name]
    sizes = ORG[name]
    rng = np.random.default_rng(len(name) + 5)
    frames = [_frame(rng, *sizes[k % len(sizes)], gray=(k % 5 == 2)) for k in range(13)]
    proto = _deploy(name, 1, *net_hw)
    one = mnet.Net(proto)
    weights = synth.make_weights(one.layers())
    one.set_params(weights)
    want = drivers.run(one, frames, spec, batch=4, net_hw=net_hw)
    assert sum(len(d) for r in want for d in r) > 0
    nets = drivers.make_nets(proto, weights, devices=[0, 0], reuse_activations=True)
    got = drivers.run(nets, frames, spec, batch=4, net_hw=net_hw)
    for i in range(len(frames)):
        for s in range(len(spec.cls_ids)):
            assert got[i][s].tobytes() == want[i][s].tobytes() and got[i][s].shape == want[i][s].shape, (i, s)
    for n in nets:
        assert set(spec.blobs) <= set(n.reuse_keep) and n.activation_misses() == 0


def test_widerface_run_over_two_reusing_nets(cuda):
    from mscnn_b200 import drivers, models, net as mnet, synth, widerface
    mnet.set_precision("fp32")
    rng = np.random.default_rng(99)
    sizes = [(120, 150), (100, 150), (130, 170), (150, 200)]
    frames = [rng.integers(0, 256, size=(*sizes[k % 4], 3), dtype=np.uint8) for k in range(10)]
    names = [f"img_{k}" for k in range(len(frames))]
    proto = models.widerface(96, 128, batch=1)
    one = mnet.Net(proto)
    weights = synth.make_weights(one.layers())
    one.set_params(weights)
    budget = 3 * 128 * 160
    want = widerface.run(one, frames, names, pixel_budget=budget)
    nets = drivers.make_nets(proto, weights, devices=[0, 0], reuse_activations=True)
    got = widerface.run(nets, frames, names, pixel_budget=budget)
    for k in names:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k
