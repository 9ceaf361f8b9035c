"""The host side of test_net_layers_gpu.py: which nets it runs, and that every layer of each of them gets exactly one
check (tests/net_layers_ref.py classify), so that a layer type or Convolution route without a check fails here.  The
fusion decisions each net is checked under (which Pooling a convolution's epilogue does, which ROIPooling writes into its
Concat, which un-pooled tops are never stored) are made when the net is built, so they are pinned here without a GPU."""
import tarfile
from collections import Counter
from pathlib import Path

import pytest

import net_layers_ref as R

ROOT = Path(__file__).resolve().parent.parent

# 23 shipped files, 18 architectures: the five -trainval files that have a sibling equal it layer for layer.  Both
# mscnn-8s-768-trainval files (KITTI car, KITTI pedestrian / cyclist) are the only 8s KITTI nets, with no other file.
SAME_AS = {
    "citypersons/mscnn-8s-1344-2x-trainval": "citypersons/mscnn-8s-1344-2x",
    "kitti_car/cascade-mscnn-7s-576-2x-trainval": "kitti_car/cascade-mscnn-7s-576-2x",
    "kitti_car/mscnn-7s-576-2x-trainval": "kitti_car/mscnn-7s-576-2x",
    "kitti_ped_cyc/mscnn-7s-576-2x-trainval": "kitti_ped_cyc/mscnn-7s-576-2x",
    "widerface/mscnn-12s-2x-trainval": "widerface/mscnn-12s-2x",
}

SIZES = [
    ("caltech-mscnn-7s-480", [(240, 320)]),
    ("caltech-mscnn-7s-480-2x", [(240, 320)]),
    ("caltech-mscnn-7s-720", [(240, 320)]),
    ("citypersons-cascade-mscnn-8s-1344-2x", [(192, 384)]),
    ("citypersons-mscnn-8s-1344-2x", [(192, 384)]),
    ("kitti_car-cascade-mscnn-7s-576-2x", [(192, 640)]),
    ("kitti_car-mscnn-7s-384", [(192, 640)]),
    ("kitti_car-mscnn-7s-384-2x", [(192, 640)]),
    ("kitti_car-mscnn-7s-576", [(192, 640)]),
    ("kitti_car-mscnn-7s-576-2x", [(192, 640)]),
    ("kitti_car-mscnn-8s-768-trainval", [(192, 640)]),
    ("kitti_ped_cyc-mscnn-7s-384", [(192, 640)]),
    ("kitti_ped_cyc-mscnn-7s-384-2x", [(192, 640)]),
    ("kitti_ped_cyc-mscnn-7s-576", [(192, 640)]),
    ("kitti_ped_cyc-mscnn-7s-576-2x", [(192, 640)]),
    ("kitti_ped_cyc-mscnn-8s-768-trainval", [(192, 640)]),
    ("widerface-cascade-mscnn-12s-align", [(128, 192)]),
    ("widerface-mscnn-12s-2x", [(128, 192)]),
    ("kitti_car-mscnn-8s-768-odd-100x324", [(100, 324)]),
    ("widerface-mscnn-12s-2x-reshaped", [(128, 192), (160, 96), (128, 192)]),
]

_TRUNK = "pool1<-conv1_2 pool2<-conv2_2 pool3<-conv3_3"
_ROI = "roi_pool_ctx<-roi_pool_org"
_ROI3 = "roi_pool_ctx<-roi_pool_org roi_pool_ctx_2nd<-roi_pool_org_2nd roi_pool_ctx_3rd<-roi_pool_org_3rd"
_STORE = "conv1_2 conv2_2 conv3_3"
_STORE_ROI = "roi_pool_ctx roi_pool_org"
_STORE_ROI3 = "roi_pool_ctx roi_pool_ctx_2nd roi_pool_ctx_3rd roi_pool_org roi_pool_org_2nd roi_pool_org_3rd"
# the routes of the Convolution and InnerProduct layers (net_layers_ref.conv_route): the KITTI car nets' square heads
# take the head taps, the rectangular heads (pedestrians) and the WIDER FACE heads the direct fp32 route
_HEAD_TAPS = "conv1_1:1 fc_f32:2 fc_planes:1 head_taps:{} planes:15"
_DIRECT = "conv1_1:1 direct_f32:{} fc_f32:2 fc_planes:1 planes:{}"
# case -> (folded layers, blobs never stored, routes)
FUSION = {
    "caltech-mscnn-7s-480": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(7, 15)),
    "caltech-mscnn-7s-480-2x": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(7, 15)),
    "caltech-mscnn-7s-720": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(7, 15)),
    "citypersons-cascade-mscnn-8s-1344-2x": (f"{_TRUNK} {_ROI3}", f"{_STORE} {_STORE_ROI3}",
                                             "conv1_1:1 direct_f32:8 fc_f32:8 fc_planes:5 planes:19"),
    "citypersons-mscnn-8s-1344-2x": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(8, 15)),
    "kitti_car-cascade-mscnn-7s-576-2x": (f"{_TRUNK} {_ROI3}", f"{_STORE} {_STORE_ROI3}",
                                          "conv1_1:1 fc_f32:6 fc_planes:3 head_taps:7 planes:17"),
    "kitti_car-mscnn-7s-384": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _HEAD_TAPS.format(7)),
    "kitti_car-mscnn-7s-384-2x": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _HEAD_TAPS.format(7)),
    "kitti_car-mscnn-7s-576": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _HEAD_TAPS.format(7)),
    "kitti_car-mscnn-7s-576-2x": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _HEAD_TAPS.format(7)),
    "kitti_car-mscnn-8s-768-trainval": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _HEAD_TAPS.format(8)),
    "kitti_ped_cyc-mscnn-7s-384": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(7, 15)),
    "kitti_ped_cyc-mscnn-7s-384-2x": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(7, 15)),
    "kitti_ped_cyc-mscnn-7s-576": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(7, 15)),
    "kitti_ped_cyc-mscnn-7s-576-2x": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(7, 15)),
    "kitti_ped_cyc-mscnn-8s-768-trainval": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(8, 15)),
    # ROIAlign then Pooling: nothing of the ROI stages is folded
    "widerface-cascade-mscnn-12s-align": (_TRUNK, _STORE, "conv1_1:1 direct_f32:12 fc_f32:8 fc_planes:5 planes:21"),
    "widerface-mscnn-12s-2x": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(12, 17)),
    # conv3_3 is 25 x 81: pool3 stays folded but conv3_3 stores its un-pooled top, and pool3 pools it itself
    "kitti_car-mscnn-8s-768-odd-100x324": (f"{_TRUNK} {_ROI}", f"conv1_2 conv2_2 {_STORE_ROI}", _HEAD_TAPS.format(8)),
    "widerface-mscnn-12s-2x-reshaped": (f"{_TRUNK} {_ROI}", f"{_STORE} {_STORE_ROI}", _DIRECT.format(12, 17)),
}


@pytest.fixture(scope="module")
def shipped(tmp_path_factory):
    d = tmp_path_factory.mktemp("deploy")
    with tarfile.open(ROOT / "tests" / "golden" / "deploy.tar.xz") as t:
        t.extractall(d, filter="data")
    return {str(f.parent.relative_to(d / "deploy")): f.read_text()
            for f in sorted((d / "deploy").glob("*/*/mscnn_deploy.prototxt"))}


def _signature(net):
    """The layer list without the input dims: every layer's parameters and parameter shapes."""
    return tuple(net.layer_param_strings()), tuple(tuple(s) for _, _, s in net.layers())


def test_architectures(shipped):
    """Files with identical layer lists once the input dims are ignored are one architecture; ARCHITECTURES holds one
    file of each."""
    from mscnn_b200.net import Net
    assert len(shipped) == 23
    groups = {}
    for key, text in shipped.items():
        groups.setdefault(_signature(Net(text)), []).append(key)
    assert len(groups) == 18, sorted(groups.values())
    rep = {}
    for keys in groups.values():
        main = [k for k in keys if k not in SAME_AS]
        assert len(main) == 1, keys
        assert sorted(keys) == sorted(main + [k for k, v in SAME_AS.items() if v == main[0]]), keys
        rep[main[0]] = keys
    assert sorted(rep) == sorted(R.ARCHITECTURES)


def test_case_list_is_pinned():
    assert [(c, s) for c, _, s in R.CASES] == SIZES
    assert sorted(FUSION) == sorted(c for c, _ in SIZES)
    assert sorted({k for _, k, _ in R.CASES}) == sorted(R.ARCHITECTURES)
    assert all(R.BATCH == 2 for _ in R.CASES)


@pytest.mark.parametrize("case", R.CASES, ids=[c[0] for c in R.CASES])
def test_every_layer_has_one_check(case):
    """Every layer of the net, at each listed size, is COMPUTE, PLANE or IDENTITY (classify raises otherwise); the
    Convolution and InnerProduct routes, the folded layers and the blobs the fused net never stores are the pinned
    ones."""
    from mscnn_b200.net import Net
    cid, key, sizes = case
    fused, unstored, routes = FUSION[cid]
    net = Net(R.deploy(key, R.BATCH, *sizes[0]))
    for h, w in sizes:
        text = R.deploy(key, R.BATCH, h, w)
        net.reshape_input("data", R.BATCH, 3, h, w)         # the reshaped case: the same net, as the GPU test runs it
        fresh = Net(text)
        for n in (net, fresh):
            classes = R.classify(n, text, key)
            assert sorted(classes) == sorted(n.layer_names)
            assert {k for k, _ in classes.values()} <= {R.COMPUTE, R.PLANE, R.IDENTITY}
            got_routes = Counter(d for name, (_, d) in classes.items()
                                 if n.layer_types[n.layer_names.index(name)] in ("Convolution", "InnerProduct"))
            assert " ".join(f"{k}:{v}" for k, v in sorted(got_routes.items())) == routes, (h, w)
            folded = sorted(f"{x}<-{n.fused_producer(x)}" for x in n.layer_names if n.fused_producer(x) != x)
            assert " ".join(folded) == fused, (h, w)
            assert " ".join(sorted(R._unstored_blobs(n))) == unstored, (h, w)
            assert n.blob_shape("data") == (R.BATCH, 3, h, w)


def test_unchecked_layers_are_refused():
    """A strided convolution on the planes route, a dense Deconvolution, a ReLU left out of its producer and a layer
    type without a check are refused, not skipped."""
    from mscnn_b200.net import Net
    head = 'name: "t"\ninput: "data" input_dim: 1 input_dim: 64 input_dim: 8 input_dim: 8\n'
    cases = [
        'layer { name: "a" type: "Convolution" bottom: "data" top: "a" convolution_param { num_output: 64 kernel_size: 3 '
        'pad: 1 stride: 2 } }',
        'layer { name: "a" type: "Deconvolution" bottom: "data" top: "a" convolution_param { num_output: 64 '
        'kernel_size: 2 stride: 2 } }',
        'layer { name: "a" type: "Convolution" bottom: "data" top: "a" convolution_param { num_output: 64 '
        'kernel_size: 3 pad: 1 } }\nlayer { name: "r" type: "ReLU" bottom: "a" top: "a" }',
    ]
    for body in cases:
        text = head + body + "\n"
        with pytest.raises(R.Unchecked):
            R.classify(Net(text), text, "kitti_car/mscnn-7s-384")
    # the library refuses a type it lacks when the net is built, so rename one of a built net's layers
    text = R.deploy("kitti_car/mscnn-7s-384", 1, 96, 320)
    net = Net(text)
    assert R.classify(net, text, "kitti_car/mscnn-7s-384")
    net.layer_types[net.layer_names.index("drop6")] = "Sigmoid"
    with pytest.raises(R.Unchecked, match="drop6: layer type Sigmoid"):
        R.classify(net, text, "kitti_car/mscnn-7s-384")


def test_prototxt_geometry_of_the_rectangular_heads(shipped):
    """kernel_h / kernel_w and pad_h / pad_w come from the prototxt text (the parameter string prints kernel_size and pad
    only): the pedestrian heads are 5x3 pad 2x1 and 7x5 pad 3x2, the parameter blobs agree."""
    from mscnn_b200.net import Net
    text = shipped["caltech/mscnn-7s-720"]
    layers = R.prototxt_layers(text)
    assert R.conv_geometry(layers["LFCN_1_3x5"]) == (5, 3, 2, 1, 1, 1, 1, 1, 1)
    assert R.conv_geometry(layers["LFCN_1_5x7"]) == (7, 5, 3, 2, 1, 1, 1, 1, 1)
    assert R.conv_geometry(layers["conv1_1"]) == (3, 3, 1, 1, 1, 1, 1, 1, 1)
    net = Net(text)
    assert net.param_shapes("LFCN_1_3x5")[0][2:] == (5, 3)
    coeffs = R.prototxt_layers(shipped["citypersons/cascade-mscnn-8s-1344-2x"])["cls_prob_3rd_avg"]
    assert coeffs["eltwise_param.coeff"] == ["0.33333333"] * 3


def test_bars():
    """The tiers of net_layers_ref.bar, from each tier's K upward."""
    assert R.bar(True, 4608) == (1e-4, 1e-4)
    assert R.bar(True, 16384) == (2e-4, 2e-4)
    assert R.bar(True, 17920) == R.bar(True, 25088) == (1e-4, 5e-4)
    assert R.bar(False, 512) == (2.0 ** -8, 1e-5)
    assert R.bar(False, 2048) == (2.0 ** -8, 2e-5)
    assert R.bar(False, 9216) == R.bar(False, 16384) == (2.0 ** -8, 1e-4)


def test_decode_bbox_restatement_matches_the_oracle():
    """decode_bbox_f32 against oracle.port.decode_bbox on random priors and predictions, with and without bbox
    normalisation: the image column exactly, each coordinate within one ulp of its exp-derived width or height plus one
    of its own (check_decode_against_port)."""
    import numpy as np
    rng = np.random.default_rng(17)
    r = 20000
    x1, y1 = rng.uniform(-50, 600, r), rng.uniform(-50, 300, r)
    prior = np.stack([rng.integers(0, 2, r), x1, y1, x1 + rng.uniform(0, 300, r), y1 + rng.uniform(0, 200, r)], 1)
    prior = prior.astype(np.float32)
    pred = rng.standard_normal((r, 8)).astype(np.float32) * 2
    for mean, std in [((0, 0, 0, 0), (1, 1, 1, 1)), ((0, 0, 0, 0), (0.1, 0.1, 0.2, 0.2))]:
        R.check_decode_against_port(R.decode_bbox_f32(pred, prior, mean, std), pred, prior, mean, std)
