"""mscnn_b200.caffe, the pycaffe surface, host only: nets are built and their parameters read and written without a
device, as in test_net_cpu.py.

For every shipped deploy net (tests/golden/deploy.tar.xz), caffe.Net gives the names net.Net gives; top_names /
bottom_names are the tops and bottoms of each layer's parameters after InsertSplits (split blobs included); params has
net.Net's shapes, and a write through a parameter's data view is what net.Net.param reads.  The refusals of a
forward-only GPU library are checked, and, where oracle/_ref is built, the layer order against the reference's own
layers."""
from __future__ import annotations

import numpy as np
import pytest

from test_layer_accesses_cpu import deploy_nets


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    return deploy_nets(tmp_path_factory.mktemp("deploy"))


def _accesses(param_string: str, key: str) -> list[str]:
    return [f[len(key):] for f in param_string.split("|") if f.startswith(key)]


def test_names_and_accesses_equal_the_net(nets):
    from mscnn_b200 import caffe, net as mnet
    splits = 0
    for rel, proto in nets.items():
        ref = mnet.Net(str(proto))
        net = caffe.Net(str(proto), caffe.TEST)
        assert net._layer_names == ref.layer_names, rel
        assert net._blob_names == ref.blob_names and list(net.blobs) == ref.blob_names, rel
        assert net.inputs == ref.inputs and net.outputs == ref.outputs, rel
        assert [l.type for l in net.layers] == ref.layer_types, rel
        assert list(net.top_names) == list(net.bottom_names) == ref.layer_names, rel
        for name, s in zip(ref.layer_names, ref.layer_param_strings()):
            assert net.bottom_names[name] == _accesses(s, "b:"), (rel, name)
            assert net.top_names[name] == _accesses(s, "t:"), (rel, name)
        splits += sum(t == "Split" for t in ref.layer_types)
        assert list(net.params) == [l for l, _, sh in ref.layers() if sh], rel
        for layer, blobs in net.params.items():
            assert [b.shape for b in blobs] == ref.param_shapes(layer), (rel, layer)
        b = net.blobs[net.inputs[0]]
        assert b.shape == ref.blob_shape(net.inputs[0]) and b.count == int(np.prod(b.shape))
        assert (b.num, b.channels, b.height, b.width) == b.shape
    assert splits > 0                       # the shipped nets do have split blobs


def test_param_view_writes_reach_the_net(nets):
    from mscnn_b200 import caffe
    net = caffe.Net(str(nets["kitti_car/mscnn-7s-576-2x"]), caffe.TEST)
    rng = np.random.default_rng(3)
    for layer in ("conv1_1", "conv4_3", "LFCN_4_5x5", "fc6", "bbox_pred"):
        for i, blob in enumerate(net.params[layer]):
            want = rng.standard_normal(blob.shape).astype(np.float32)
            blob.data[...] = want
            assert np.array_equal(net.mscnn_net.param(layer, i), want), (layer, i)
            assert np.array_equal(net.params[layer][i].data, want), (layer, i)   # a fresh view of the same bytes


def test_constructor_forms_and_refusals(nets, tmp_path):
    from mscnn_b200 import caffe, capi
    proto = str(nets["kitti_car/mscnn-7s-384"])
    with pytest.raises(capi.MscnnError, match="forward-only"):
        caffe.Net(proto, caffe.TRAIN)
    with pytest.raises(capi.MscnnError, match="Could not open file"):
        caffe.Net(str(tmp_path / "missing.prototxt"), caffe.TEST)
    with pytest.raises(capi.MscnnError, match="Could not open file"):
        caffe.Net(proto, str(tmp_path / "missing.caffemodel"), caffe.TEST)
    with pytest.raises(capi.MscnnError, match="Could not open file"):
        caffe.Net(proto, caffe.TEST, weights=str(tmp_path / "missing.caffemodel"))
    with pytest.raises(capi.MscnnError, match="GPU only"):
        caffe.set_mode_cpu()
    caffe.set_mode_gpu()
    net = caffe.Net(proto, caffe.TEST)
    with pytest.raises(AttributeError, match="forward-only"):
        net.blobs["data"].diff
    with pytest.raises(AttributeError, match="forward-only"):
        net.params["conv1_1"][0].diff
    with pytest.raises(capi.MscnnError, match="do not match net inputs"):
        net.forward(conv1_1=np.zeros((1, 64, 384, 1280), np.float32))
    with pytest.raises(capi.MscnnError, match="not batch sized"):
        net.forward(data=np.zeros((2, 3, 384, 1280), np.float32))
    with pytest.raises(capi.MscnnError, match="N x C x H x W"):
        net.blobs["data"].reshape(3, 384, 1280)


def test_layer_type_list():
    from mscnn_b200 import caffe
    types = caffe.layer_type_list()
    assert types == sorted(types)
    assert {"Input", "Convolution", "Pooling", "ReLU", "Split", "Concat", "BoxOutput", "ROIPooling", "InnerProduct",
            "Softmax", "Deconvolution", "DecodeBBox"} <= set(types)
    assert "MemoryData" not in types and "Python" not in types


def test_layer_order_equals_the_reference(nets):
    """The reference's own layers (oracle/_ref, built where the reference sources are) read each deploy net in the
    prototxt's layer order; the net inserts its split layers between them (InsertSplits) and keeps that order."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref is not built")
    from mscnn_b200 import caffe
    for rel, proto in nets.items():
        net = caffe.Net(str(proto), caffe.TEST)
        r = ref.RefNet(str(proto), is_path=True)
        assert [l for l, lr in zip(net._layer_names, net.layers) if lr.type != "Split"] == r.layer_names, rel
        assert [lr.type for lr in net.layers if lr.type != "Split"] == r.layer_types, rel
        for b in net._blob_names:
            if "_split_" not in b:
                r.blob_shape(b)                 # raises KeyError for a blob the reference does not make
        for layer, blobs in net.params.items():
            assert [b.shape for b in blobs] == r.param_shapes(layer), (rel, layer)
