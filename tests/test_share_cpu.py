"""Nets that share their trained parameters, and the drivers' hand-out of batches to several nets, host side (no GPU).

(a) Net.share_trained_layers_with (Net::ShareTrainedLayersWith, net.cpp:682-712): parameters are matched by layer name,
    layers the target lacks are ignored, a blob count or shape mismatch is refused with the reference's message and
    shares nothing; afterwards a write through either net shows in the other's param(), and the ParamSpec-name sharing
    inside each net keeps working.
(b) Precision and stream are per host thread in Python as they are in the library.
(c) drivers.serve_batches on fake nets: whole batches in input order from one queue, each exactly once; results by
    image index equal the one-net results whatever the interleaving (uneven last batches, WIDER buckets); a worker
    that raises stops the hand-out, every thread is joined and the exception reaches the caller."""
import random
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def _conv_net(layers):
    """A net of 3x3 convolutions on an 8-channel 6x6 input: layers = [(name, num_output, bias_term)], chained."""
    s = 'input: "d" input_dim: 1 input_dim: 8 input_dim: 6 input_dim: 6\n'
    bottom = "d"
    for name, cout, bias in layers:
        s += (f'layer {{ name: "{name}" type: "Convolution" bottom: "{bottom}" top: "{name}" convolution_param {{ '
              f'num_output: {cout} kernel_size: 3 pad: 1 bias_term: {"true" if bias else "false"} '
              f'weight_filler {{ type: "gaussian" std: 0.1 }} }} }}\n')
        bottom = name
    return s


def _fill(net, seed):
    rng = np.random.default_rng(seed)
    w = {n: [rng.standard_normal(s).astype(np.float32) for s in shp] for n, _, shp in net.layers() if shp}
    net.set_params(w)
    return w


def test_share_matches_layers_by_name_and_ignores_missing_ones():
    from mscnn_b200.net import Net
    src = Net(_conv_net([("a", 16, True), ("b", 16, True), ("only_src", 8, False)]))
    dst = Net(_conv_net([("a", 16, True), ("b", 16, True), ("only_dst", 8, True)]))
    ws = _fill(src, 1)
    wd = _fill(dst, 2)
    dst.share_trained_layers_with(src)
    for layer in ("a", "b"):
        for j in range(2):
            assert np.array_equal(dst.param(layer, j), ws[layer][j]), (layer, j)
    for j in range(2):                                   # a layer the source lacks keeps its own parameters
        assert np.array_equal(dst.param("only_dst", j), wd["only_dst"][j])
    assert np.array_equal(src.param("only_src", 0), ws["only_src"][0])

    # writes through either net show in both
    new = np.full(ws["b"][0].shape, 0.5, np.float32)
    dst.set_params({"b": [new]})
    assert np.array_equal(src.param("b", 0), new)
    bias = np.arange(16, dtype=np.float32)
    src.set_params({"a": [ws["a"][0], bias]})
    assert np.array_equal(dst.param("a", 1), bias)
    assert np.array_equal(dst.param("b", 1), ws["b"][1])   # the other blob of the layer is untouched


def test_share_keeps_param_name_sharing_inside_each_net():
    from mscnn_b200 import models
    from mscnn_b200.net import Net
    a, b = Net(models.widerface_cascade(128, 192)), Net(models.widerface_cascade(128, 192))
    b.share_trained_layers_with(a)
    w = np.full(a.param_shapes("cls_pred")[0], 0.25, dtype=np.float32)
    b.set_params({"cls_pred": [w, np.arange(2, dtype=np.float32)]})
    for net in (a, b):                              # cls_pred_1st_3rd shares cls_pred's blobs by ParamSpec name
        assert np.array_equal(net.param("cls_pred", 0), w)
        assert np.array_equal(net.param("cls_pred_1st_3rd", 0), w)
        assert np.array_equal(net.param("cls_pred_1st_3rd", 1), [0, 1])
    a.set_params({"cls_pred_2nd_3rd": [2 * w, np.zeros(2, dtype=np.float32)]})
    assert np.array_equal(b.param("cls_pred_2nd", 0), 2 * w)


_SHARE = ("import sys\nfrom mscnn_b200 import capi\nfrom mscnn_b200.net import Net\n"
          "src, dst = Net(sys.argv[1]), Net(sys.argv[2])\n"
          "before = dst.param('b', 0).copy()\n"
          "try:\n    dst.share_trained_layers_with(src)\nexcept capi.MscnnError:\n    print('refused')\n"
          "print('unchanged' if (dst.param('b', 0) == before).all() else 'changed')\n")


@pytest.mark.parametrize("src_layers,message", [
    ([("a", 16, True), ("b", 16, False)], "Incompatible number of blobs for layer b"),
    ([("a", 16, True), ("b", 24, True)], "Cannot share param 0 weights from layer 'b'; shape mismatch.  Source param "
                                         "shape is 24 16 3 3 (3456); target param shape is 16 16 3 3 (2304)"),
])
def test_share_refuses_count_and_shape_mismatches(src_layers, message):
    """The reference's CHECK messages, on stderr; the C entry returns MSCNN_ERR_INVALID and shares nothing (the
    matching layer 'a' before the bad one keeps its own blobs too)."""
    src = _conv_net(src_layers)
    dst = _conv_net([("a", 16, True), ("b", 16, True)])
    r = subprocess.run([sys.executable, "-c", _SHARE, src, dst], capture_output=True, text=True, cwd=str(ROOT))
    assert r.returncode == 0, r.stderr[-600:]
    assert r.stdout.split() == ["refused", "unchanged"], r.stdout
    assert message in r.stderr, r.stderr[-600:]


def test_share_refusal_shares_nothing_in_process():
    from mscnn_b200 import capi
    from mscnn_b200.net import Net
    src = Net(_conv_net([("a", 16, True), ("b", 24, True)]))
    dst = Net(_conv_net([("a", 16, True), ("b", 16, True)]))
    _fill(src, 3)
    wd = _fill(dst, 4)
    with pytest.raises(capi.MscnnError):
        dst.share_trained_layers_with(src)
    src.set_params({"a": [np.zeros((16, 8, 3, 3), np.float32), np.zeros(16, np.float32)]})
    assert np.array_equal(dst.param("a", 0), wd["a"][0])


def test_precision_and_stream_are_per_thread():
    from mscnn_b200 import net as mnet
    mnet.set_precision("fp32")
    seen = {}

    def other():
        seen["initial"] = (mnet.get_precision(), getattr(mnet._local, "stream_ptr", None))
        mnet.set_precision("bf16")
        mnet.set_stream(0x1000)              # recorded only: no CUDA call is made
        seen["set"] = (mnet.get_precision(), mnet._local.stream_ptr)
        mnet.set_stream(None)

    mnet.set_stream(None)
    t = threading.Thread(target=other)
    t.start()
    t.join()
    assert seen["initial"] == ("fp32", None) and seen["set"] == ("bf16", 0x1000)
    assert mnet.get_precision() == "fp32" and getattr(mnet._local, "stream_ptr", None) is None


# ------------------------------------------------------------------------------------- (c) batches over several nets
class _FakeNet:
    def __init__(self, k, fail_on=None):
        self.k, self.fail_on, self.batches, self.thread = k, fail_on, [], None


def _results(batches, nets, seed, out, log):
    """serve_batches over fake nets whose 'forward' of a batch takes a random time and writes f(i) for every image."""
    from mscnn_b200 import drivers
    rng = random.Random(seed)
    delays = {id(n): [rng.uniform(0, 0.004) for _ in range(64)] for n in nets}

    def handed_out():                       # runs inside take(), so `log` is the hand-out order
        for b in batches:
            log.append(tuple(b[1] if isinstance(b, tuple) else b))
            yield b

    def serve(net, take):
        net.thread = threading.current_thread().name
        b = take()
        while b is not None:
            if net.fail_on is not None and len(net.batches) == net.fail_on:
                raise RuntimeError(f"net {net.k} failed")
            time.sleep(delays[id(net)][len(net.batches) % 64])
            for i in (b[1] if isinstance(b, tuple) else b):
                out[i] = (i * 7 + 3, b[0] if isinstance(b, tuple) else len(b))
            net.batches.append(b)
            b = take()

    drivers.serve_batches(nets, handed_out(), serve)


@pytest.mark.parametrize("n_frames,batch,n_nets", [(20, 8, 2), (33, 4, 3), (3, 8, 4), (16, 8, 1), (41, 5, 8)])
def test_fixed_size_batches_over_fake_nets(n_frames, batch, n_nets):
    chunks = [list(range(k, min(k + batch, n_frames))) for k in range(0, n_frames, batch)]
    want = [(i * 7 + 3, len(c)) for c in chunks for i in c]
    for seed in range(3):
        nets = [_FakeNet(k) for k in range(n_nets)]
        out, log = [None] * n_frames, []
        _results(chunks, nets, seed, out, log)
        assert out == want, seed
        assert log == [tuple(c) for c in chunks]                     # handed out whole, in input order, once each
        assert sorted(tuple(b) for n in nets for b in n.batches) == sorted(tuple(c) for c in chunks)
        used = [n for n in nets if n.batches]
        assert len({n.thread for n in used}) == len(used)             # one thread per net
        assert threading.current_thread().name not in {n.thread for n in used}


def test_wider_buckets_over_fake_nets():
    from mscnn_b200 import widerface
    rng = np.random.default_rng(7)
    hw = [(int(rng.integers(80, 1600)), int(rng.integers(80, 1600))) for _ in range(32)]
    batches = widerface.plan_batches(hw, max_batch=4, pixel_budget=4 * 512 * 512)
    want = [None] * len(hw)
    for net_hw, idx in batches:
        for i in idx:
            want[i] = (i * 7 + 3, net_hw)
    for seed in range(3):
        nets = [_FakeNet(k) for k in range(3)]
        out, log = [None] * len(hw), []
        _results(batches, nets, seed, out, log)
        assert out == want
        assert log == [tuple(idx) for _, idx in batches]            # largest net size first, as plan_batches orders


def test_a_failing_worker_stops_the_others():
    from mscnn_b200 import drivers
    chunks = [list(range(k, k + 2)) for k in range(0, 200, 2)]
    before = {t.name for t in threading.enumerate()}
    nets = [_FakeNet(0), _FakeNet(1, fail_on=2), _FakeNet(2)]
    out, log = [None] * 200, []
    with pytest.raises(RuntimeError, match="net 1 failed"):
        _results(chunks, nets, 0, out, log)
    assert not [t for t in threading.enumerate() if t.name.startswith("mscnn-net-") and t.name not in before]
    assert len(log) < len(chunks)

    # once a worker has raised, take() hands out nothing more
    after = []

    def serve(net, take):
        if net.k == 0:
            take()
            raise KeyError("first batch")
        time.sleep(0.3)
        after.append(take())

    with pytest.raises(KeyError):
        drivers.serve_batches([_FakeNet(0), _FakeNet(1), _FakeNet(2)], chunks, serve)
    assert after == [None, None]
    with pytest.raises(ValueError):
        drivers.serve_batches([nets[0], nets[0]], chunks, lambda n, t: None)


def test_run_over_fake_nets_equals_one_net(monkeypatch):
    """drivers.run with a list: the same chunks as one net, each served on its net's thread, merged by image index."""
    import contextlib
    from mscnn_b200 import drivers
    frames = [np.zeros((5 + i % 3, 7, 3), np.uint8) for i in range(21)]
    calls = []

    def fake_serve(net, take, frames_, spec, net_hw, pre, out):
        b = take()
        while b is not None:
            calls.append((net if isinstance(net, _FakeNet) else None, tuple(b)))
            for i in b:
                out[i] = [np.full((1, 5), i, np.float32)]
            b = take()

    monkeypatch.setattr(drivers, "_serve_fixed", fake_serve)
    monkeypatch.setattr(drivers, "net_thread", lambda net, precision: contextlib.nullcontext())
    one = drivers.run("one net", frames, drivers.KITTI_CAR, batch=8)
    nets = [_FakeNet(0), _FakeNet(1)]
    many = drivers.run(nets, frames, drivers.KITTI_CAR, batch=8)
    assert [r[0].tobytes() for r in one] == [r[0].tobytes() for r in many]
    assert sorted(b for n, b in calls if n is not None) == [tuple(range(0, 8)), tuple(range(8, 16)),
                                                            tuple(range(16, 21))]
    with pytest.raises(ValueError):
        drivers.run(nets, frames, drivers.KITTI_CAR, pre=["only one plan"])
