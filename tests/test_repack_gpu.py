"""A live Net re-packs the weights and biases its kernels read exactly when it has to: after a parameter update, a
precision switch or a change of the LFCN head route (MSCNN_NO_HEAD_TAPS with a config reload), and never from stale
buffers.  One net goes through every step; after each step it must compute, bit for bit, what a net built afresh with
the same parameters and settings computes: every output, the LFCN maps, the proposal counts and the final detections.

The nets cover every packing route: conv1_1, trunk convolutions with fused pooling, the LFCN heads on the tap route
(k x k) or the generic one (1 x 1, or every head under MSCNN_NO_HEAD_TAPS), and the InnerProduct layers; the WIDER
cascade's third stage shares fc6 and cls_pred with the first stage by parameter name."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# kind: (net args, two LFCN heads, whether its heads take the tap route)
NETS = {
    "kitti8s": ((96, 320, 8, False), ("LFCN_1_5x5", "LFCN_2_7x7"), True),
    "kitti_cascade": ((96, 320), ("LFCN_1_5x5", "LFCN_3_7x7"), True),
    "wider_cascade": ((128, 192), ("LFCN_1_12x12", "LFCN_2_64x64"), False),
}


def _set_param(net, layer, idx, a):
    """Write one parameter blob, leaving the layer's other blobs (and their versions) alone."""
    from mscnn_b200 import capi
    a = np.ascontiguousarray(a, dtype=np.float32)
    capi.check(net._L.mscnn_net_set_param(net._h, layer.encode(), idx, a.ctypes.data, a.size), f"set_param({layer})")


def _detections(cuda, net, kind, h, w):
    from mscnn_b200 import capi, net as mnet
    if kind == "kitti8s":
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
    if kind == "kitti8s":
        net.detect(cfg, dets.data_ptr(), cnt.data_ptr())
    else:
        net.detect_cascade(cfg, dets.data_ptr(), cnt.data_ptr(), stage="3rd",
                           cls_prob=None if kind == "kitti_cascade" else "cls_prob_3rd_avg")
    torch.cuda.synchronize()
    return dets.cpu().numpy(), cnt.cpu().numpy()


def _run(cuda, net, kind, h, w, images):
    res = dict(net.forward(data=images))
    res.update({n: net.blob(n) for n in net.layer_names if n.startswith("LFCN") or n == "cls_pred"})
    res["num_proposals"] = np.array([net.num_proposals(), net.num_proposals(0), net.num_proposals(1)])
    res["detections"], res["detection_counts"] = _detections(cuda, net, kind, h, w)
    return res


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _assert_same(got, want, step):
    assert sorted(got) == sorted(want), step
    for k in want:
        assert _same(got[k], want[k]), (step, k)


@pytest.mark.parametrize("kind", list(NETS))
def test_live_net_repacks_like_a_fresh_net(cuda, kind, monkeypatch):
    from mscnn_b200 import models, net as mnet, ops, synth
    args, heads, tap_heads = NETS[kind]
    h, w = args[0], args[1]
    proto = getattr(models, "kitti" if kind == "kitti8s" else kind.replace("wider", "widerface"))(*args, batch=2)
    images = synth.make_images(2, h, w)
    updates = []          # (layer, blob index, values) written after the base parameters

    def fresh():
        net = mnet.Net(proto)
        net.set_params(base)
        for u in updates:
            _set_param(net, *u)
        return _run(cuda, net, kind, h, w, images)

    def step(name):
        got = _run(cuda, live, kind, h, w, images)
        _assert_same(got, fresh(), name)
        return got

    try:
        mnet.set_precision("fp32")
        live = mnet.Net(proto)
        base = synth.make_weights(live.layers())
        live.set_params(base)
        assert live.fused_producer("pool3") == "conv3_3"
        first = step("fp32")
        assert first["num_proposals"][0] > 0
        mnet.set_precision("bf16")
        step("bf16")
        mnet.set_precision("fp32")
        _assert_same(_run(cuda, live, kind, h, w, images), first, "fp32 again")

        for layer in ("conv1_1", "conv3_3", heads[0], "fc6"):
            updates.append((layer, 0, base[layer][0] * np.float32(0.9)))
        for layer in ("cls_pred", heads[1]):
            updates.append((layer, 1, base[layer][1] + np.float32(0.25)))
        for u in updates:
            _set_param(live, *u)
        updated = step("updated parameters")
        assert not _same(updated["cls_pred"], first["cls_pred"])

        monkeypatch.setenv("MSCNN_NO_HEAD_TAPS", "1")
        ops.reload_config()
        direct = step("MSCNN_NO_HEAD_TAPS=1")
        if tap_heads:       # the route really changed: the two head formulations sum in different orders
            assert any(not _same(direct[n], updated[n]) for n in direct if n.startswith("LFCN"))
        monkeypatch.delenv("MSCNN_NO_HEAD_TAPS")
        ops.reload_config()
        step("head taps again")
    finally:
        monkeypatch.delenv("MSCNN_NO_HEAD_TAPS", raising=False)
        ops.reload_config()
        mnet.set_precision("fp32")
