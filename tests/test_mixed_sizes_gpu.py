"""Batches of images with different ORIGINAL sizes on the device.  The reference drivers read each frame's size inside
their loop and rescale / clip its detections with that frame's ratios (examples/kitti_car/run_mscnn_detection.m:64-65,
:111-116; run_cascademscnn.m:77-80, :101-105); here one batch carries N sizes:
  * pre-processing: every slot of a mixed batch == oracle.port.preprocess of its image, bit for bit;
  * post-process: the hand-derived vectors as one batch, and slot n of a sized call == the cfg entry called with image
    n's geometry, bit for bit, on real net outputs (plain, packed, cascade, single-rank push);
  * Net: set_input_images(list) -> forward -> detect, geometry belongs to the forward (pipelined order, graph replay)."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import port

pytestmark = pytest.mark.gpu

CASES = json.loads((Path(__file__).resolve().parent / "golden" / "a15_postprocess_cases.json").read_text())["cases"]
KITTI = [(375, 1242), (370, 1224), (374, 1238), (376, 1241)]


def _frames(rng, sizes):
    out = []
    for h, w in sizes:
        im = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        im[: h // 3, : w // 3] = 255             # saturating overshoot region
        out.append(im)
    return out


def _ref(frames, out_hw):
    return np.stack([port.preprocess(im, out_hw) for im in frames])


# ------------------------------------------------------------------------------------------------ pre-processing
def test_preprocess_mixed_sizes_bit_exact(cuda):
    from mscnn_b200 import ops
    out_hw = (384, 1280)
    # KITTI-like upscales, an antialiased downscale, an identity, and two images whose pass order differs
    # (100 x 1400: width pass first; 1400 x 100: height pass first)
    sizes = KITTI + [(600, 2000), (384, 1280), (100, 1400), (1400, 100)]
    rng = np.random.default_rng(17)
    frames = _frames(rng, sizes)
    pre = ops.Preprocess(KITTI[0], out_hw)
    ref = _ref(frames, out_hw)
    got_host = pre(frames).cpu().numpy()
    got_dev = pre([torch.from_numpy(f).cuda() for f in frames]).cpu().numpy()
    for n in range(len(sizes)):
        assert np.array_equal(got_host[n], ref[n]), sizes[n]
        assert np.array_equal(got_dev[n], ref[n]), sizes[n]
    # a new mix: cached and new sizes, in another order
    sizes2 = [(200, 700), KITTI[2], (384, 1280), (500, 1500), KITTI[0]]
    frames2 = _frames(rng, sizes2)
    assert np.array_equal(pre(frames2).cpu().numpy(), _ref(frames2, out_hw))
    assert np.array_equal(pre([torch.from_numpy(f).cuda() for f in frames2]).cpu().numpy(), _ref(frames2, out_hw))
    # a uniform batch through the sized entry == the array entry
    uni = _frames(rng, [KITTI[0]] * 3)
    arr = np.stack(uni)
    assert torch.equal(pre(uni), pre(arr))
    assert torch.equal(pre([torch.from_numpy(f).cuda() for f in uni]), pre(torch.from_numpy(arr).cuda()))


def test_preprocess_more_images_than_one_launch(cuda):
    """70 images: the descriptors of one launch hold 32, so the batch takes three launches of each pass."""
    from mscnn_b200 import ops
    rng = np.random.default_rng(5)
    sizes = [(int(rng.integers(5, 60)), int(rng.integers(5, 60))) for _ in range(70)]
    frames = _frames(rng, sizes)
    pre = ops.Preprocess(sizes[0], (24, 40))
    got = pre(frames).cpu().numpy()
    assert np.array_equal(got, _ref(frames, (24, 40)))


# -------------------------------------------------------------------------------- hand-derived post-process vectors
def _batch_cfg(num_cls):
    from mscnn_b200 import capi
    cfg = capi.DetectCfg()
    cfg.num_cls, cfg.cls_id = num_cls, 2
    for k, v in enumerate([0.1, 0.1, 0.2, 0.2]):
        cfg.bbox_std[k], cfg.bbox_mean[k] = v, 0.0
    cfg.proposal_thr, cfg.nms_overlap = -10.0, 0.5
    cfg.ratio_h, cfg.ratio_w, cfg.org_h, cfg.org_w = 7.0, 7.0, 3.0, 3.0     # ignored by the sized entries
    cfg.max_rois_per_image = 64
    return cfg


def _num_out(counts, cuda):
    t = int(sum(counts))
    return torch.tensor([max(t, 1), t] + list(counts), dtype=torch.int32, device=cuda)


def _case_geometry(c):
    oh, ow = c.get("org_hw", c["net_hw"])
    return [c["ratios"][0], c["ratios"][1], oh, ow]


@pytest.mark.parametrize("repeat", [1, 24])
def test_postprocess_hand_vectors_as_one_batch(cuda, repeat):
    """The three `postprocess` cases (5 classes, three geometries) as one batch; repeat = 24 gives 72 images, more than
    the 64 geometries one launch carries."""
    from mscnn_b200 import ops
    cases = [c for c in CASES if c["kind"] == "postprocess"] * repeat
    cat = lambda k: torch.from_numpy(np.concatenate([np.array(c[k], np.float32) for c in cases])).to(cuda)
    geo = np.array([_case_geometry(c) for c in cases], np.float32)
    dets, cnt = ops.detect_postprocess(_batch_cfg(5), len(cases), cat("proposals_score"), cat("cls_pred"),
                                       cat("bbox_pred"), _num_out([len(c["proposals_score"]) for c in cases], cuda),
                                       geometry=geo)
    torch.cuda.synchronize()
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    for n, c in enumerate(cases):
        want = np.array(c["dets"], np.float64)
        assert cnt[n] == len(want), (n, c["name"])
        np.testing.assert_allclose(dets[n, :cnt[n]], want, rtol=c["tol"], atol=c["tol"], err_msg=c["name"])


def test_cascade_hand_vectors_as_one_batch(cuda):
    from mscnn_b200 import ops
    cases = [c for c in CASES if c["kind"] == "cascade"]
    cat = lambda k: torch.from_numpy(np.concatenate([np.array(c[k], np.float32) for c in cases])).to(cuda)
    geo = np.array([_case_geometry(c) for c in cases], np.float32)
    dets, cnt = ops.cascade_detect_postprocess(_batch_cfg(2), len(cases), cat("proposals"), cat("cls_prob"),
                                               cat("output_bbox"), _num_out([len(c["proposals"]) for c in cases], cuda),
                                               geometry=geo)
    torch.cuda.synchronize()
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    for n, c in enumerate(cases):
        want = np.array(c["dets"], np.float64)
        assert cnt[n] == len(want), (n, c["name"])
        np.testing.assert_allclose(dets[n, :cnt[n]], want, rtol=c["tol"], atol=c["tol"], err_msg=c["name"])


# ------------------------------------------------------------------------- sized == uniform on real net outputs
ORG_4 = [(375, 1242), (370, 1224), (188, 621), (96, 320)]


def _kitti_net(h, w, b, cascade=False):
    from mscnn_b200 import models, net as mnet, synth
    mnet.set_precision("fp32")
    proto = models.kitti_cascade(h, w, batch=b) if cascade else models.kitti(h, w, 8, False, batch=b)
    net = mnet.Net(proto)
    net.set_params(synth.make_weights(net.layers()))
    return net


def _net_rows(net, b, cuda):
    return _num_out([net.num_proposals(i) for i in range(b)], cuda)


def _blob(net, name, cuda):
    return torch.from_numpy(net.blob(name)).to(cuda)


def _assert_slots_equal(dets, cnt, per_image):
    """per_image[n] = (dets, counts) of a cfg-entry call: slot n must match bit for bit."""
    for n, (d, c) in enumerate(per_image):
        assert int(cnt[n]) == int(c[n]), n
        assert torch.equal(dets[n, :int(cnt[n])], d[n, :int(c[n])]), n


def test_sized_equals_uniform_on_net_outputs(cuda):
    from mscnn_b200 import capi, net as mnet, ops, parallel, synth
    h, w, b = 192, 640, 4
    net = _kitti_net(h, w, b)
    net.forward(data=synth.make_images(b, h, w))
    ps, cp, bp = (_blob(net, k, cuda) for k in ("proposals_score", "cls_pred", "bbox_pred"))
    num_out = _net_rows(net, b, cuda)
    cfg = mnet.kitti_detect_cfg(h, w)
    geo = mnet.image_geometry((h, w), ORG_4)
    dets, cnt = ops.detect_postprocess(cfg, b, ps, cp, bp, num_out, geometry=geo)
    per_image = [ops.detect_postprocess(mnet.kitti_detect_cfg(h, w, org_hw=o), b, ps, cp, bp, num_out) for o in ORG_4]
    torch.cuda.synchronize()
    assert int(cnt.sum()) > 0
    _assert_slots_equal(dets, cnt, per_image)
    # packed form
    import ctypes as C
    cap = cfg.max_rois_per_image
    nbytes = C.c_size_t(0)
    L = capi.lib()
    capi.check(L.mscnn_detect_workspace_bytes(cfg, b, C.byref(nbytes)), "ws")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=cuda)
    payload = torch.zeros(parallel.payload_floats(b, cap), device=cuda)
    capi.check(L.mscnn_detect_postprocess_packed_sized(cfg, b, capi.ptr(ps), capi.ptr(cp), capi.ptr(bp),
                                                       capi.ptr(num_out), capi.ptr(ws), nbytes.value, capi.ptr(payload),
                                                       geo.ctypes.data, ops._stream()), "packed_sized")
    torch.cuda.synchronize()
    got = parallel.unpack_payload(payload, 1, b, cap)
    d, c = dets.cpu().numpy(), cnt.cpu().numpy()
    for n in range(b):
        assert np.array_equal(got[n], d[n, :c[n]]), n


def test_cascade_sized_equals_uniform_on_net_outputs(cuda):
    from mscnn_b200 import net as mnet, ops, synth
    h, w, b = 96, 320, 4
    net = _kitti_net(h, w, b, cascade=True)
    net.forward(data=synth.make_images(b, h, w))
    pr, cl, ob = (_blob(net, k, cuda) for k in ("proposals_3rd", "cls_prob_3rd", "output_bbox_3rd"))
    num_out = _net_rows(net, b, cuda)
    cfg = mnet.kitti_detect_cfg(h, w)
    geo = mnet.image_geometry((h, w), ORG_4)
    dets, cnt = ops.cascade_detect_postprocess(cfg, b, pr, cl, ob, num_out, geometry=geo)
    per_image = [ops.cascade_detect_postprocess(mnet.kitti_detect_cfg(h, w, org_hw=o), b, pr, cl, ob, num_out)
                 for o in ORG_4]
    torch.cuda.synchronize()
    assert int(cnt.sum()) > 0
    _assert_slots_equal(dets, cnt, per_image)
    # the Net facade's cascade entry with the geometry of the forward
    net.set_input_geometry(ORG_4)
    net.forward_only()
    d2 = torch.zeros_like(dets)
    c2 = torch.zeros_like(cnt)
    net.detect_cascade(cfg, d2.data_ptr(), c2.data_ptr(), stage="3rd")
    torch.cuda.synchronize()
    assert torch.equal(c2, cnt) and torch.equal(d2, dets)


def test_detect_push_single_rank_uses_forward_geometry(cuda):
    from mscnn_b200 import net as mnet, ops, parallel, synth
    mnet.set_stream(torch.cuda.current_stream().cuda_stream)
    h, w, b = 192, 640, 4
    net = _kitti_net(h, w, b)
    net.set_input("data", synth.make_images(b, h, w, first_index=3))
    net.set_input_geometry(ORG_4)
    net.forward_only()
    cfg = mnet.kitti_detect_cfg(h, w)
    cap = cfg.max_rois_per_image
    x = parallel.PeerExchange(b, cap, rank=0, world=1, generations=2)
    net.detect_push(cfg, x)
    x.wait(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = parallel.unpack_payload(x.gathered(), 1, b, cap)
    dets, cnt = ops.detect_postprocess(cfg, b, *(_blob(net, k, cuda) for k in ("proposals_score", "cls_pred",
                                                                                 "bbox_pred")),
                                       _net_rows(net, b, cuda), geometry=mnet.image_geometry((h, w), ORG_4))
    torch.cuda.synchronize()
    d, c = dets.cpu().numpy(), cnt.cpu().numpy()
    assert int(c.sum()) > 0
    for n in range(b):
        assert np.array_equal(got[n], d[n, :c[n]]), n
    x.close()


# ------------------------------------------------------------------------------------------------- Net end to end
H, W, B = 192, 640, 4
SIZES_A = KITTI
SIZES_B = [(370, 1224), (512, 1700), (375, 1242), (300, 1000)]


def _detect(net, cuda, cfg=None):
    from mscnn_b200 import net as mnet
    cfg = cfg or mnet.kitti_detect_cfg(H, W)
    dets = torch.zeros((B, cfg.max_rois_per_image, 5), device=cuda)
    cnt = torch.zeros(B, dtype=torch.int32, device=cuda)
    net.detect(cfg, dets.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    return dets, cnt


def _post(net, cuda, sizes):
    from mscnn_b200 import net as mnet, ops
    args = [_blob(net, k, cuda) for k in ("proposals_score", "cls_pred", "bbox_pred")] + [_net_rows(net, B, cuda)]
    geo = None if sizes is None else mnet.image_geometry((H, W), sizes)
    out = ops.detect_postprocess(mnet.kitti_detect_cfg(H, W), B, *args, geometry=geo)
    torch.cuda.synchronize()
    return out


def test_net_mixed_frames_end_to_end(cuda):
    from mscnn_b200 import ops
    net = _kitti_net(H, W, B)
    frames = _frames(np.random.default_rng(3), SIZES_A)
    pre = ops.Preprocess(SIZES_A[0], (H, W))
    net.set_input_images("data", pre, frames)
    net.forward_only()
    assert np.array_equal(net.blob("data"), _ref(frames, (H, W)))
    dets, cnt = _detect(net, cuda)
    want = _post(net, cuda, SIZES_A)
    assert int(cnt.sum()) > 0 and torch.equal(cnt, want[1]) and torch.equal(dets, want[0])
    d, c = dets.cpu().numpy(), cnt.cpu().numpy()
    for n, (oh, ow) in enumerate(SIZES_A):
        k = d[n, :c[n]]
        assert np.all(k[:, 0] >= 0) and np.all(k[:, 1] >= 0)
        assert np.all(k[:, 0] + k[:, 2] <= ow * (1 + 1e-6)) and np.all(k[:, 1] + k[:, 3] <= oh * (1 + 1e-6)), n


def test_geometry_belongs_to_the_forward(cuda):
    from mscnn_b200 import net as mnet, ops
    rng = np.random.default_rng(9)
    fa, fb = _frames(rng, SIZES_A), _frames(rng, SIZES_B)
    pre = ops.Preprocess(SIZES_A[0], (H, W))
    net = _kitti_net(H, W, B)
    want = {}
    for key, frames, sizes in (("a", fa, SIZES_A), ("b", fb, SIZES_B)):
        net.set_input_images("data", pre, frames)
        net.forward_only()
        want[key] = _detect(net, cuda)
        ref = _post(net, cuda, sizes)
        assert torch.equal(want[key][0], ref[0]) and torch.equal(want[key][1], ref[1])
    assert not torch.equal(want["a"][0], want["b"][0])
    # pipelined order: set the next batch, then detect the current one
    net.set_input_images("data", pre, fa)
    net.forward_only()
    net.set_input_images("data", pre, fb)
    got = _detect(net, cuda)
    assert torch.equal(got[0], want["a"][0]) and torch.equal(got[1], want["a"][1])
    net.forward_only()
    got = _detect(net, cuda)
    assert torch.equal(got[0], want["b"][0]) and torch.equal(got[1], want["b"][1])
    # a forward without recorded sizes is back on the cfg's scalars
    net.set_input("data", net.blob("data"))
    net.forward_only()
    cfg = mnet.kitti_detect_cfg(H, W, org_hw=(300, 1000))
    got = _detect(net, cuda, cfg)
    ref = ops.detect_postprocess(cfg, B, *(_blob(net, k, cuda) for k in ("proposals_score", "cls_pred", "bbox_pred")),
                                 _net_rows(net, B, cuda))
    torch.cuda.synchronize()
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    # set_input_geometry alone, with a caller-filled input; a count that does not match the batch is refused
    net.set_input_geometry(SIZES_B)
    net.forward_only()
    got = _detect(net, cuda)
    ref = _post(net, cuda, SIZES_B)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    net.set_input_geometry(SIZES_B[:2])
    with pytest.raises(Exception):
        net.forward_only()
    net.set_input_geometry(None)


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


def test_graph_replay_with_mixed_sizes(side_stream, cuda):
    from mscnn_b200 import ops
    rng = np.random.default_rng(21)
    fa, fb = _frames(rng, SIZES_A), _frames(rng, SIZES_B)
    pre = ops.Preprocess(SIZES_A[0], (H, W))
    eager = _kitti_net(H, W, B)
    want = []
    for frames in (fa, fb):
        eager.set_input_images("data", pre, frames)
        eager.forward_only()
        want.append(_detect(eager, cuda))
    net = _kitti_net(H, W, B)
    net.set_graph(True)
    replays = 0
    for which in (0, 1, 0, 1):
        net.set_input_images("data", pre, (fa, fb)[which])
        net.forward_only()
        replays += int(net.graph_replayed())
        got = _detect(net, cuda)
        assert torch.equal(got[0], want[which][0]) and torch.equal(got[1], want[which][1]), which
    assert replays >= 2
