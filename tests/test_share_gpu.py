"""Nets that share one copy of the weights, and the drivers over several nets, on the GPU.

(a) A second KITTI net that shares the first's weights grows device memory on its first forward by its activations
    only, a weight's worth less than a second net with weights of its own, and packs no weight image.
(b) Both sharing nets compute, bit for bit, what one net computes: fp32-faithful and bf16, eager and CUDA graph.
(c) A weight written through net B is what net A computes with next, after exactly one re-pack; A's graph is dropped.
(d) Forwards of the two nets from two host threads, each on its own stream, equal the sequential run.
(e) drivers.run over [net, sharing net] (KITTI car, KITTI cascade) and widerface.run over mixed sizes equal the one-net
    runs bit for bit, gray frames included; then across two devices when there are two."""
import threading

import numpy as np
import pytest
import torch

from test_drivers_gpu import NET_HW, ORG, _deploy, _frame

pytestmark = pytest.mark.gpu


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


def _packs():
    from mscnn_b200 import capi, net as mnet
    L = capi.lib()
    mnet._declare(L)
    return int(L.mscnn_weight_pack_count())


def _kitti(batch=2, h=96, w=320):
    from mscnn_b200 import models
    return models.kitti(h, w, 8, False, batch=batch)


def _outputs(net, images):
    out = net.forward(data=images)
    out["num_proposals"] = np.array([net.num_proposals()])
    return out


def _assert_same(got, want, step):
    assert sorted(got) == sorted(want), step
    for k in want:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), (step, k)


def _set_param(net, layer, idx, a):
    from mscnn_b200 import capi
    a = np.ascontiguousarray(a, dtype=np.float32)
    capi.check(net._L.mscnn_net_set_param(net._h, layer.encode(), idx, a.ctypes.data, a.size), f"set_param({layer})")


def test_second_net_allocates_no_weight_memory(cuda):
    from mscnn_b200 import net as mnet, synth
    mnet.set_precision("fp32")
    proto = _kitti(batch=2, h=192, w=640)
    images = synth.make_images(2, 192, 640)
    a = mnet.Net(proto)
    weights = synth.make_weights(a.layers())
    a.set_params(weights)
    want = _outputs(a, images)
    torch.cuda.synchronize()
    weight_bytes = 4 * sum(int(np.prod(s)) for _, _, shp in a.layers() for s in shp)

    def first_forward(make):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        p0 = _packs()
        net = make()
        got = _outputs(net, images)
        torch.cuda.synchronize()
        return net, got, free0 - torch.cuda.mem_get_info()[0], _packs() - p0

    def shared():
        b = mnet.Net(proto)
        b.share_trained_layers_with(a)
        return b

    def own():
        c = mnet.Net(proto)
        c.set_params(weights)
        return c

    b, got_b, grow_shared, packs_shared = first_forward(shared)
    c, got_c, grow_own, packs_own = first_forward(own)
    _assert_same(got_b, want, "shared")
    _assert_same(got_c, want, "own")
    assert packs_shared == 0 and packs_own > 0, (packs_shared, packs_own)
    # the own-weights net holds fp32 weights and their packed hi / lo images (about twice the fp32 bytes) on top
    assert grow_own - grow_shared >= 1.5 * weight_bytes, (grow_own, grow_shared, weight_bytes)
    print(f"weights {weight_bytes / 2**20:.1f} MiB; first forward: sharing net +{grow_shared / 2**20:.1f} MiB, "
          f"own weights +{grow_own / 2**20:.1f} MiB")


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sharing_nets_equal_one_net(request, cuda, precision, graph):
    from mscnn_b200 import net as mnet, synth
    if graph:
        request.getfixturevalue("side_stream")
    mnet.set_precision(precision)
    try:
        proto = _kitti()
        batches = [synth.make_images(2, 96, 320, first_index=2 * s) for s in (1, 2, 3)]
        ref = mnet.Net(proto)
        weights = synth.make_weights(ref.layers())
        ref.set_params(weights)
        want = [_outputs(ref, x) for x in batches]
        del ref
        a = mnet.Net(proto)
        a.set_params(weights)
        b = mnet.Net(proto)
        b.share_trained_layers_with(a)
        for net in (a, b):
            net.set_graph(graph)
        replays = 0
        for rnd in range(2):
            for k, x in enumerate(batches):
                for name, net in (("a", a), ("b", b)):
                    _assert_same(_outputs(net, x), want[k], (rnd, k, name))
                    replays += int(net.graph_replayed())
        if graph:
            assert replays >= 6, replays
    finally:
        mnet.set_precision("fp32")


@pytest.mark.parametrize("graph", [False, True])
def test_write_through_one_net_reaches_the_other(request, cuda, graph):
    from mscnn_b200 import net as mnet, synth
    if graph:
        request.getfixturevalue("side_stream")
    mnet.set_precision("fp32")
    proto = _kitti()
    images = synth.make_images(2, 96, 320)
    a = mnet.Net(proto)
    weights = synth.make_weights(a.layers())
    a.set_params(weights)
    b = mnet.Net(proto)
    b.share_trained_layers_with(a)
    a.set_graph(graph)
    first = _outputs(a, images)
    _outputs(a, images)
    _outputs(b, images)
    assert a.graph_replayed() == graph

    new = weights["conv3_3"][0] * np.float32(0.9)
    fresh = mnet.Net(proto)
    fresh.set_params(weights)
    _set_param(fresh, "conv3_3", 0, new)
    want = _outputs(fresh, images)
    del fresh
    assert not np.array_equal(want["cls_pred"], first["cls_pred"])

    _set_param(b, "conv3_3", 0, new)
    p0 = _packs()
    _assert_same(_outputs(a, images), want, "A after a write through B")
    assert not a.graph_replayed()
    _assert_same(_outputs(b, images), want, "B after its own write")
    assert _packs() - p0 == 1                     # conv3_3's image, packed once for both nets
    if graph:
        _outputs(a, images)
        _assert_same(_outputs(a, images), want, "A replayed")
        assert a.graph_replayed()
    assert np.array_equal(a.param("conv3_3", 0), new)


def test_two_threads_equal_the_sequential_run(cuda):
    from mscnn_b200 import net as mnet, synth
    mnet.set_precision("fp32")
    proto = _kitti()
    batches = [synth.make_images(2, 96, 320, first_index=2 * s) for s in range(6)]
    ref = mnet.Net(proto)
    weights = synth.make_weights(ref.layers())
    ref.set_params(weights)
    want = [_outputs(ref, x) for x in batches]
    del ref
    a = mnet.Net(proto)
    a.set_params(weights)
    b = mnet.Net(proto)
    b.share_trained_layers_with(a)
    got = {}
    errors = []

    def worker(net, name, order):
        try:
            s = torch.cuda.Stream()
            mnet.set_stream(s.cuda_stream)
            mnet.set_precision("fp32")
            with torch.cuda.stream(s):
                for rnd in range(2):
                    for k in order:
                        got[(name, rnd, k)] = _outputs(net, batches[k])
            s.synchronize()
            mnet.set_stream(None)
        except BaseException as e:     # noqa: BLE001 -- reported below
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(a, "a", range(6))),
               threading.Thread(target=worker, args=(b, "b", range(5, -1, -1)))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert len(got) == 24
    for (name, rnd, k), out in got.items():
        _assert_same(out, want[k], (name, rnd, k))


@pytest.mark.parametrize("name", ["kitti_car", "kitti_car_cascade"])
def test_driver_run_over_two_sharing_nets(cuda, name):
    from mscnn_b200 import drivers, net as mnet, synth
    mnet.set_precision("fp32")
    spec = drivers.SPECS[name]
    net_hw = NET_HW[name]
    sizes = ORG["kitti_car"]
    rng = np.random.default_rng(len(name) + 1)
    frames = [_frame(rng, *sizes[k % len(sizes)], gray=(k % 5 == 2)) for k in range(21)]
    frames[7] = frames[7][:, :, :1] if frames[7].ndim == 3 else frames[7][:, :, None]
    proto = _deploy(name, 1, *net_hw)
    one = mnet.Net(proto)
    weights = synth.make_weights(one.layers())
    one.set_params(weights)
    want = drivers.run(one, frames, spec, batch=4, net_hw=net_hw)        # batches of 4, the last one short
    assert sum(len(d) for r in want for d in r) > 0
    nets = drivers.make_nets(proto, weights, devices=[0, 0])
    for _ in range(2):
        got = drivers.run(nets, frames, spec, batch=4, net_hw=net_hw)
        assert len(got) == len(frames)
        for i in range(len(frames)):
            for s in range(len(spec.cls_ids)):
                assert got[i][s].tobytes() == want[i][s].tobytes() and got[i][s].shape == want[i][s].shape, (i, s)
    # the caller's net, stream and precision are untouched: one net on this thread still gives the same result
    again = drivers.run(nets[0], frames, spec, batch=4, net_hw=net_hw)
    assert all(a[0].tobytes() == b[0].tobytes() for a, b in zip(again, want))


def test_driver_error_in_a_worker_reaches_the_caller(cuda):
    from mscnn_b200 import drivers, net as mnet, synth
    proto = _deploy("kitti_car", 1, *NET_HW["kitti_car"])
    one = mnet.Net(proto)
    nets = drivers.make_nets(proto, synth.make_weights(one.layers()), devices=[0, 0])
    rng = np.random.default_rng(3)
    frames = [_frame(rng, 120, 400) for _ in range(8)]
    before = threading.active_count()
    from mscnn_b200 import ops
    bad = [ops.Preprocess((120, 400), (96, 320)) for _ in nets]      # not the net size: the first batch raises
    with pytest.raises(ValueError, match="pre-processing plan"):
        drivers.run(nets, frames, drivers.KITTI_CAR, batch=2, net_hw=NET_HW["kitti_car"], pre=bad)
    assert threading.active_count() == before


def test_widerface_run_over_two_sharing_nets(cuda):
    from mscnn_b200 import drivers, models, net as mnet, synth, widerface
    mnet.set_precision("fp32")
    rng = np.random.default_rng(2025)
    sizes = [(120, 150), (100, 150), (130, 170), (150, 200), (90, 130)]
    frames = []
    for k in range(12):
        h, w = sizes[k % len(sizes)]
        im = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        im[: h // 4, : w // 4] = 255
        frames.append(im)
    names = [f"img_{k}" for k in range(len(frames))]
    proto = models.widerface(96, 128, batch=1)
    one = mnet.Net(proto)
    weights = synth.make_weights(one.layers())
    one.set_params(weights)
    budget = 3 * 128 * 160
    want = widerface.run(one, frames, names, pixel_budget=budget)
    assert sum(len(v) for v in want.values()) > 0
    nets = drivers.make_nets(proto, weights, devices=[0, 0])
    got = widerface.run(nets, frames, names, pixel_budget=budget)
    assert list(got) == names
    for k in names:
        assert got[k].shape == want[k].shape and got[k].tobytes() == want[k].tobytes(), k


def test_nets_on_two_devices(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two devices")
    from mscnn_b200 import capi, drivers, net as mnet, synth
    mnet.set_precision("fp32")
    spec = drivers.KITTI_CAR
    net_hw = NET_HW["kitti_car"]
    proto = _deploy("kitti_car", 1, *net_hw)
    one = mnet.Net(proto)
    weights = synth.make_weights(one.layers())
    one.set_params(weights)
    rng = np.random.default_rng(9)
    frames = [_frame(rng, *ORG["kitti_car"][k % 4], gray=(k % 4 == 1)) for k in range(24)]
    want = drivers.run(one, frames, spec, batch=4, net_hw=net_hw)
    nets = drivers.make_nets(proto, weights, devices=[0, 1, 1])
    assert [n.device for n in nets] == [0, 1, 1] and torch.cuda.current_device() == 0
    with pytest.raises(capi.MscnnError):
        nets[1].share_trained_layers_with(nets[0])            # across devices: refused
    got = drivers.run(nets, frames, spec, batch=4, net_hw=net_hw)
    for i in range(len(frames)):
        assert got[i][0].tobytes() == want[i][0].tobytes(), i
