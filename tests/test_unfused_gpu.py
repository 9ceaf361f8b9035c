"""The unfused layer path (MSCNN_NO_FUSION=1: stand-alone ReLU, Concat and un-pooled convolutions) and the host-synced
row path (MSCNN_SYNC_ROWS=1: every layer behind BoxOutput sized to the exact R instead of the cap) compute what the
default, fused and device-count Net computes, bit for bit.

Why identity and not a tolerance: mscnn_relu_planes zeroes (hi, lo) exactly when hi < 0, so it commutes with the
split of max(x, 0); Concat copies bytes; ROIPooling is per row; a convolution row sums its K terms in an order the layer
fixes, whatever pixel box the M dimension is tiled with (and SYNC_ROWS changes the head's N, so possibly the box)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _split(x):
    """fp32 -> (hi, lo) bf16 planes, hi = bf16(x), lo = bf16(x - hi)."""
    hi = x.bfloat16()
    return hi, (x - hi.float()).bfloat16()


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _relu_inputs():
    g = torch.Generator(device="cpu").manual_seed(71)
    x = torch.randn((3, 5, 7, 64), generator=g) * 4.0
    flat = x.view(-1)
    tiny = torch.tensor([1e-39, -1e-39, 3e-40, -3e-40, 1.2e-38, -1.2e-38, 1e-45, -1e-45])   # fp32 / bf16 denormals
    flat[:8] = tiny
    flat[8:16] = torch.tensor([-0.0, 0.0, -0.0, 0.0, -1.0, 1.0, -2.0 ** -130, 2.0 ** -130])
    # values whose lo has the opposite sign to hi: hi rounds away from zero
    flat[16:24] = torch.tensor([1 + 2.0 ** -8 + 2.0 ** -10, -(1 + 2.0 ** -8 + 2.0 ** -10), 3.9999, -3.9999,
                                 1e-38 * 1.999, -1e-38 * 1.999, 255.9, -255.9])
    hi, lo = _split(x)
    assert bool(((hi.float() * lo.float()) < 0).any()) and bool((lo.float() != 0).any())
    return x


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_relu_planes(cuda, split):
    """mscnn_relu_planes == the split of max(x, 0), bit for bit, in place."""
    from mscnn_b200 import capi
    x = _relu_inputs()
    hi, lo = _split(x)
    if split:
        ref_hi, ref_lo = _split(torch.where(x > 0, x, torch.zeros_like(x)))
    else:
        ref_hi = torch.where(hi.float() > 0, hi, torch.zeros_like(hi))
    d_hi = hi.to(cuda)
    d_lo = lo.to(cuda) if split else None
    capi.check(capi.lib().mscnn_relu_planes(capi.ptr(d_hi), capi.ptr(d_lo), d_hi.numel(),
                                            torch.cuda.current_stream().cuda_stream), "relu_planes")
    torch.cuda.synchronize()
    assert torch.equal(_bits(d_hi.cpu()), _bits(ref_hi))
    if split:
        assert torch.equal(_bits(d_lo.cpu()), _bits(ref_lo))


def test_relu_f32(cuda):
    from mscnn_b200 import capi
    x = _relu_inputs().view(-1)[:1000].clone()          # not a multiple of 8: the fp32 entry takes any count
    d = x.to(cuda)
    capi.check(capi.lib().mscnn_relu_f32(capi.ptr(d), d.numel(), torch.cuda.current_stream().cuda_stream), "relu_f32")
    torch.cuda.synchronize()
    got = d.cpu()
    ref = torch.where(x > 0, x, torch.zeros_like(x))
    assert torch.equal(got, ref)                        # -0 and +0 compare equal: max(-0, 0) may be either
    assert bool((got[x < 0] == 0).all()) and torch.equal(_bits(got[x > 0]), _bits(x[x > 0]))


@pytest.mark.parametrize("offsets", [(0, 64), (128, 0), (8, 200), (192, 64, 264)])
def test_concat_planes(cuda, offsets):
    """mscnn_concat_planes at several offsets == torch.cat, the channels no input covers untouched."""
    from mscnn_b200 import capi
    g = torch.Generator(device="cpu").manual_seed(73)
    pixels = 2 * 9 * 13
    widths = [64, 72, 128][: len(offsets)]
    ctot = max(o + c for o, c in zip(offsets, widths)) + 8
    xs = [torch.randn((pixels, c), generator=g).bfloat16().to(cuda) for c in widths]
    y = torch.full((pixels, ctot), 0x7FBF, dtype=torch.int16, device=cuda).view(torch.bfloat16)
    ref = y.clone()
    for o, x in zip(offsets, xs):
        ref[:, o:o + x.shape[1]] = x
        capi.check(capi.lib().mscnn_concat_planes(capi.ptr(x), capi.ptr(y), pixels, x.shape[1], ctot, o,
                                                  torch.cuda.current_stream().cuda_stream), "concat_planes")
    torch.cuda.synchronize()
    assert torch.equal(_bits(y), _bits(ref))
    order = sorted(range(len(offsets)), key=lambda i: offsets[i])
    if all(offsets[order[i]] + widths[order[i]] == offsets[order[i + 1]] for i in range(len(order) - 1)):
        lo = offsets[order[0]]
        cat = torch.cat([xs[i] for i in order], dim=1)
        assert torch.equal(_bits(y[:, lo:lo + cat.shape[1]]), _bits(cat))


# ------------------------------------------------------------------------------------------------------ Net level
def _layer_io(net):
    io = {}
    for s in net.layer_param_strings():
        parts = s.split("|")
        io[parts[0]] = ([p[2:] for p in parts if p.startswith("b:")], [p[2:] for p in parts if p.startswith("t:")])
    return io


def _unstored_blobs(net):
    """Blobs the fused net never writes: the un-pooled output of a convolution whose pooling runs in its epilogue (at
    even extents; at odd ones the convolution stores it and the Pooling runs itself), and the tops of ROIPooling layers
    that write straight into their Concat's output."""
    io = _layer_io(net)
    skip = set()
    for name, typ in zip(net.layer_names, net.layer_types):
        prod = net.fused_producer(name)
        if prod == name:
            continue
        if typ == "Pooling":
            bottom = io[name][0][0]
            if all(e % 2 == 0 for e in net.blob_shape(bottom)[2:]):
                skip.add(bottom)
        elif typ == "ROIPooling":
            skip.update(io[name][1])
            skip.update(io[prod][1])
    return skip


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


NETS = [
    ("kitti8s_fp32", "kitti", (192, 640, 8, False), "fp32"),
    ("kitti8s_bf16", "kitti", (192, 640, 8, False), "bf16"),
    # conv3_3 is 25 x 81: pool3 runs itself, pool1 and pool2 stay in their convolutions' epilogues
    ("kitti8s_odd", "kitti", (100, 324, 8, False), "fp32"),
    ("kitti7s_2x", "kitti", (96, 320, 7, True), "fp32"),
    ("kitti_cascade", "kitti_cascade", (96, 320), "fp32"),
    ("wider_cascade", "widerface_cascade", (128, 192), "fp32"),
]


def _detections(cuda, net, kind, h, w):
    from mscnn_b200 import capi, net as mnet
    if kind == "kitti":
        cfg = mnet.kitti_detect_cfg(h, w)
    else:
        cfg = capi.DetectCfg()
        cfg.num_cls, cfg.cls_id = (5, 2) if kind == "kitti_cascade" else (2, 2)
        cfg.nms_overlap = 0.5 if kind == "kitti_cascade" else 0.3
        cfg.ratio_h, cfg.ratio_w = 1.25, 0.8
        cfg.org_h, cfg.org_w = h / 1.25, w / 0.8
        cfg.max_rois_per_image = 3000
    dets = torch.zeros((2, cfg.max_rois_per_image, 5), device=cuda)
    cnt = torch.zeros(2, dtype=torch.int32, device=cuda)
    if kind == "kitti":
        net.detect(cfg, dets.data_ptr(), cnt.data_ptr())
    else:
        net.detect_cascade(cfg, dets.data_ptr(), cnt.data_ptr(), stage="3rd",
                           cls_prob=None if kind == "kitti_cascade" else "cls_prob_3rd_avg")
    torch.cuda.synchronize()
    return dets.cpu().numpy(), cnt.cpu().numpy()


@pytest.mark.parametrize("case", NETS, ids=[c[0] for c in NETS])
def test_unfused_and_synced_nets_are_bit_identical(cuda, case, monkeypatch):
    from mscnn_b200 import models, net as mnet, synth
    _, kind, args, precision = case
    h, w = args[0], args[1]
    proto = getattr(models, kind)(*args, batch=2)
    mnet.set_precision(precision)
    nets = {}
    for variant, env in [("default", None), ("MSCNN_NO_FUSION", "MSCNN_NO_FUSION"), ("MSCNN_SYNC_ROWS", "MSCNN_SYNC_ROWS")]:
        with monkeypatch.context() as m:
            if env:
                m.setenv(env, "1")
            nets[variant] = mnet.Net(proto)          # the switches are read when the net is built
    weights = synth.make_weights(nets["default"].layers())
    images = synth.make_images(2, h, w)
    outs, props, dets = {}, {}, {}
    for variant, net in nets.items():
        net.set_params(weights)
        outs[variant] = net.forward(data=images)
        props[variant] = [net.num_proposals(i) for i in range(2)]
        dets[variant] = _detections(cuda, net, kind, h, w)
    base = nets["default"]
    skip = _unstored_blobs(base)
    assert not _unstored_blobs(nets["MSCNN_NO_FUSION"])
    if (h, w) == (100, 324):
        assert base.fused_producer("pool3") == "conv3_3" and "conv3_3" not in skip
        assert {"conv1_2", "conv2_2"} <= skip
    assert sum(props["default"]) > 0
    for variant in ("MSCNN_NO_FUSION", "MSCNN_SYNC_ROWS"):
        net = nets[variant]
        assert props[variant] == props["default"], variant
        assert sorted(outs[variant]) == sorted(outs["default"])
        for k in outs["default"]:
            assert _same(outs[variant][k], outs["default"][k]), (variant, "output", k)
        for a, b in zip(dets[variant], dets["default"]):
            assert _same(a, b), (variant, "detections")
        assert net.blob_names == base.blob_names
        compared = 0
        for name in base.blob_names:
            if name in skip:
                continue
            assert _same(net.blob(name), base.blob(name)), (variant, "blob", name)
            compared += 1
        assert compared > 20, compared
