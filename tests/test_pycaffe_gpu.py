"""mscnn_b200.caffe on the device: code written the pycaffe way gives what the library's own entries give.

* A KITTI loop ported the way a pycaffe user ports run_mscnn_detection.m: ops.Preprocess output written into
  blobs['data'].data, forward(), then the driver's numpy post-process (detect_classes_ref.py) on the data views of
  proposals_score, cls_pred and bbox_pred.  Every image's detections equal drivers.run's bit for bit, in both
  precisions.
* The data views: an input written after a forward is read by the next one; a weight written through params[...].data
  gives the outputs of a net given the changed weights by set_params; blobs['data'].reshape then reshape() runs at the
  new size.
* forward(start=, end=) equals net.Net.forward_only over the same range; forward_all pads the last batch.
* share_with packs no weight again; with activation reuse on, a kept blob reads and a released one raises."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_drivers_gpu import ORG, _deploy, _frame

pytestmark = pytest.mark.gpu

NET_HW = (192, 640)


def _proto(tmp_path, n=1, hw=NET_HW, name="kitti_car"):
    p = tmp_path / f"{name}_{n}x{hw[0]}x{hw[1]}.prototxt"
    p.write_text(_deploy(name, n, *hw))
    return str(p)


def _load(net, weights):
    """The weights written the pycaffe way, through each parameter's data view."""
    for layer, blobs in net.params.items():
        for i, b in enumerate(blobs):
            b.data[...] = weights[layer][i]


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.fixture(scope="module")
def weights():
    from mscnn_b200 import net as mnet, synth
    return synth.make_weights(mnet.Net(_deploy("kitti_car", 1, *NET_HW)).layers())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_pycaffe_kitti_loop_equals_drivers_run(cuda, tmp_path, weights, precision):
    import detect_classes_ref as R
    from mscnn_b200 import caffe, drivers, net as mnet, ops
    mnet.set_precision(precision)
    try:
        spec = drivers.SPECS["kitti_car"]
        rng = np.random.default_rng(11)
        frames = [_frame(rng, *ORG["kitti_car"][k % 4]) for k in range(6)]
        net = caffe.Net(_proto(tmp_path), caffe.TEST)
        _load(net, weights)
        got = []
        for im in frames:                                  # run_mscnn_detection.m:59-120, one image per forward
            oh, ow = im.shape[:2]
            net.blobs["data"].data[...] = ops.Preprocess((oh, ow), NET_HW)(im[None]).cpu().numpy()
            net.forward()
            got.append(R.detect_postprocess_classes(
                net.blobs["proposals_score"].data, net.blobs["cls_pred"].data, net.blobs["bbox_pred"].data,
                spec.cls_ids, det_thr=spec.det_thr, bbox_std=spec.bbox_stds, proposal_thr=spec.proposal_thr,
                overlap=spec.nms_overlap, ratios=(NET_HW[0] / oh, NET_HW[1] / ow), org_hw=(oh, ow)))
        ref = mnet.Net(_deploy("kitti_car", 1, *NET_HW))
        ref.set_params(weights)
        want = drivers.run(ref, frames, spec, batch=4, net_hw=NET_HW)
        assert sum(len(d) for r in want for d in r) > 0
        for i in range(len(frames)):
            assert len(got[i]) == len(want[i]) == 1
            assert _same(got[i][0], want[i][0]), (i, got[i][0].shape, want[i][0].shape)
    finally:
        mnet.set_precision("fp32")


def test_views_inputs_weights_and_reshape(cuda, tmp_path, weights):
    from mscnn_b200 import caffe, net as mnet, synth
    mnet.set_precision("fp32")
    net = caffe.Net(_proto(tmp_path), caffe.TEST)
    _load(net, weights)
    ref = mnet.Net(_deploy("kitti_car", 1, *NET_HW))
    ref.set_params(weights)
    x1, x2 = synth.make_images(1, *NET_HW), synth.make_images(1, *NET_HW, first_index=5)
    seen = []
    for x in (x1, x2):                                     # the second write lands after the first forward
        net.blobs["data"].data[...] = x
        net.forward()
        seen.append(net.blobs["conv4_3"].data.copy())
        ref.forward(data=x)
        assert _same(seen[-1], ref.blob("conv4_3"))
    assert not _same(seen[0], seen[1])

    w = net.params["conv4_3"][0].data                      # one view, written in place
    w *= np.float32(0.5)
    out = net.forward(blobs=["conv4_3"])
    changed = {k: [b.copy() for b in v] for k, v in weights.items()}
    changed["conv4_3"][0] = changed["conv4_3"][0] * np.float32(0.5)
    fresh = mnet.Net(_deploy("kitti_car", 1, *NET_HW))
    fresh.set_params(changed)
    want = fresh.forward(data=x2)
    for k in ref.outputs:
        assert _same(out[k], want[k]), k
    assert _same(out["conv4_3"], fresh.blob("conv4_3")) and not _same(out["conv4_3"], seen[1])

    x3 = synth.make_images(2, 160, 512)
    net.blobs["data"].reshape(2, 3, 160, 512)
    net.reshape()
    assert net.blobs["conv4_3"].shape[0] == 2 and net.blobs["data"].data.shape == (2, 3, 160, 512)
    net.blobs["data"].data[...] = x3
    net.forward()
    fresh.forward(data=x3)
    for k in ("conv4_3",) + tuple(ref.outputs):
        assert _same(net.blobs[k].data, fresh.blob(k)), k


def test_partial_forward_and_forward_all(cuda, tmp_path, weights):
    from mscnn_b200 import caffe, net as mnet, synth
    mnet.set_precision("fp32")
    net = caffe.Net(_proto(tmp_path), caffe.TEST)
    _load(net, weights)
    ref = mnet.Net(_deploy("kitti_car", 1, *NET_HW))
    ref.set_params(weights)
    x = synth.make_images(1, *NET_HW)
    out = net.forward(end="conv3_3", data=x)
    ref.set_input("data", x)
    ref.forward_only(end="conv3_3")
    assert list(out) == ["conv3_3"] and _same(out["conv3_3"], ref.blob("conv3_3"))
    out = net.forward(start="conv4_1", end="conv4_3")
    ref.forward_only("conv4_1", "conv4_3")
    assert _same(out["conv4_3"], ref.blob("conv4_3"))

    # forward_all on a net whose outputs have one row per image: 11 images at batch 8 = two forwards, the second
    # padded with three zero images, cut back to 11 rows
    small = tmp_path / "small.prototxt"
    small.write_text('layer { name: "input" type: "Input" top: "data" input_param { shape { dim: 8 dim: 64 dim: 16 '
                     'dim: 16 } } }\n'
                     'layer { name: "conv" type: "Convolution" bottom: "data" top: "conv" '
                     'convolution_param { num_output: 64 kernel_size: 3 pad: 1 } }\n'
                     'layer { name: "relu" type: "ReLU" bottom: "conv" top: "conv" }\n'
                     'layer { name: "pool" type: "Pooling" bottom: "conv" top: "pool" '
                     'pooling_param { pool: MAX kernel_size: 2 stride: 2 } }\n')
    net = caffe.Net(str(small), caffe.TEST)
    rng = np.random.default_rng(5)
    net.params["conv"][0].data[...] = rng.standard_normal(net.params["conv"][0].shape).astype(np.float32) * 0.05
    net.params["conv"][1].data[...] = rng.standard_normal(64).astype(np.float32)
    xs = rng.standard_normal((11, 64, 16, 16)).astype(np.float32)
    got = net.forward_all(data=xs)
    a = net.forward(data=xs[:8])["pool"]
    b = net.forward(data=np.concatenate([xs[8:], np.zeros((5, 64, 16, 16), np.float32)]))["pool"]
    assert list(got) == ["pool"] and got["pool"].shape == (11, 64, 8, 8)
    assert _same(got["pool"], np.concatenate([a, b[:3]]))


def test_share_with_and_activation_reuse(cuda, tmp_path, weights):
    from mscnn_b200 import caffe, capi, net as mnet, synth
    mnet.set_precision("fp32")
    L = capi.lib()
    mnet._declare(L)
    x = synth.make_images(1, *NET_HW)
    a = caffe.Net(_proto(tmp_path), caffe.TEST)
    _load(a, weights)
    want = a.forward(blobs=["conv4_3"], data=x)
    packs = L.mscnn_weight_pack_count()
    b = caffe.Net(_proto(tmp_path), caffe.TEST)
    b.share_with(a)
    got = b.forward(blobs=["conv4_3"], data=x)
    assert L.mscnn_weight_pack_count() == packs
    for k in want:
        assert _same(got[k], want[k]), k

    b.mscnn_net.set_activation_reuse(True, keep=["conv4_3"])
    out = b.forward(data=x)
    assert _same(b.blobs["conv4_3"].data, want["conv4_3"])
    for k in b.outputs:
        assert _same(out[k], want[k]) and _same(b.blobs[k].data, want[k]), k
    with pytest.raises(capi.MscnnError, match="conv1_1"):
        b.blobs["conv1_1"].data
    assert b.mscnn_net.activation_misses() == 0
