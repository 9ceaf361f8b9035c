"""The nets of the Caltech and CityPersons drivers (caltech/mscnn-7s-720, citypersons/cascade-mscnn-8s-1344-2x) and the
single-stage CityPersons net (citypersons/mscnn-8s-1344-2x) against the reference's own layers, fp32-faithful:

* end to end against golden vectors from oracle/_ref (tests/golden/make_pedestrian_golden.py), at the bars of the
  KITTI nets (test_net_gpu.py): trunk, every LFCN map, the proposals row by row and the heads on aligned rows;
* the detection stages fed with the reference's own feature map and proposals (live oracle/_ref), so that no discrete
  decision upstream differs and rows line up one to one;
* the final detections of the drivers' post-process (Caltech without bbox normalisation, CityPersons on the Eltwise
  average cls_prob_3rd_avg) against the restated MATLAB post-process on the net's own outputs.

These nets are the only ones with 1:2 anchors, 5x3 / 7x5 heads and 8x4 ROI bins; a swap of h and w anywhere in them
keeps every shape consistent, so only values can show it."""
import re
import tarfile
from pathlib import Path

import numpy as np
import pytest
import torch

from test_net_gpu import _build, _check_rows_and_head, _match_rows, _rel_ok, _stage_rows

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
SUB = 7919
HEAD_KERNELS = {"3x5": (5, 3), "5x7": (7, 5)}     # LFCN_<i>_<kw>x<kh>: kernel_h x kernel_w


def _deploy(net, n, h, w):
    """The shipped deploy file deploy/<net> with its input set to n x 3 x h x w."""
    with tarfile.open(GOLD / "deploy.tar.xz") as t:
        text = t.extractfile(f"deploy/{net}/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: \d+\s+input_dim: \d+",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def _check_trunk_and_heads(net, g, trunk, nheads):
    """Sub-sampled trunk blobs and every LFCN map: >= 99.9 % within 1e-3; the heads are 6-channel maps of the
    rectangular kernels."""
    worst = {}
    for b in trunk:
        x = net.blob(b)
        assert tuple(g[b + "__shape"]) == x.shape, b
        sub, ref, m2 = x.reshape(-1)[::SUB], g[b + "__sub"], float(g[b + "__m2"][0])
        worst[b] = float(_rel_ok(sub, ref, 1e-3, m2).mean())
        assert worst[b] >= 0.999, (b, worst[b])
    heads = [k for k in g.files if k.startswith("LFCN_")]
    assert len(heads) == nheads
    for b in heads:
        x, ref = net.blob(b), g[b]
        assert x.shape == ref.shape and x.shape[1] == 6, (b, x.shape)
        assert net.param_shapes(b)[0][2:] == HEAD_KERNELS[b[-3:]], (b, net.param_shapes(b))
        m2 = float(np.mean(ref.astype(np.float64) ** 2))
        worst[b] = float(_rel_ok(x, ref, 1e-3, m2).mean())
        assert worst[b] >= 0.999, (b, worst[b])
    print("fraction within 1e-3:", worst)


def _cfg(spec, h, w, org_hw):
    """The driver's post-process settings at net size h x w for an original image of org_hw."""
    from mscnn_b200 import net as mnet
    cfg, classes = spec.detect_cfg((h, w))
    geo = mnet.kitti_detect_cfg(h, w, org_hw=org_hw)
    cfg.ratio_h, cfg.ratio_w, cfg.org_h, cfg.org_w = geo.ratio_h, geo.ratio_w, geo.org_h, geo.org_w
    return cfg, classes


# ------------------------------------------------------------------------------------------------------ end to end
def test_e2e_caltech_vs_reference_and_detect_classes(cuda):
    """caltech/mscnn-7s-720 at 2x3x240x320: seven heads on 1:2 anchors, BoxOutput without bbox normalisation, 8x4 ROI
    pooling at 1/8 on conv4_3.  Then Net.detect_classes with the Caltech driver's settings (do_bb_norm = 0) against the
    restated post-process with bbox_std 1 on the net's own outputs."""
    import detect_classes_ref as R
    from mscnn_b200 import drivers
    g = np.load(GOLD / "e2e_caltech_7s_240x320.npz")
    n, h, w = 2, 240, 320
    net = _build(_deploy("caltech/mscnn-7s-720", n, h, w), n, h, w)
    net.forward_only()
    _check_trunk_and_heads(net, g, ["conv4_3", "conv5_3", "conv6_1"], 7)
    out = {k: net.blob(k) for k in ("proposals_score", "cls_pred", "bbox_pred")}
    assert out["cls_pred"].shape[1] == 2 and out["bbox_pred"].shape[1] == 8
    assert net.blob("roi_pool").shape[1:] == (1024, 8, 4)
    _check_rows_and_head(out, g, 1e-3, 0.997, 0.99, 0.98, "caltech 7s 240x320")

    cfg, classes = _cfg(drivers.CALTECH, h, w, (480, 640))
    assert list(cfg.bbox_std) == [1.0] * 4 and list(cfg.bbox_mean) == [0.0] * 4
    dets = torch.zeros((n, 1, cfg.max_rois_per_image, 5), device=cuda)
    cnt = torch.zeros((n, 1), dtype=torch.int32, device=cuda)
    net.detect_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    ps = out["proposals_score"].reshape(-1, 6)
    start = 0
    for i in range(n):
        sl = slice(start, start + net.num_proposals(i))
        ref, = R.detect_postprocess_classes(ps[sl], out["cls_pred"][sl], out["bbox_pred"][sl], [2],
                                            bbox_mean=(0, 0, 0, 0), bbox_std=(1, 1, 1, 1),
                                            ratios=(cfg.ratio_h, cfg.ratio_w), org_hw=(cfg.org_h, cfg.org_w))
        assert cnt[i, 0] == len(ref), (i, cnt[i, 0], len(ref))
        np.testing.assert_allclose(dets[i, 0, :cnt[i, 0]], ref, rtol=1e-5, atol=1e-5)
        start = sl.stop
    assert start == len(ps) and cnt.sum() > 0
    print(f"caltech: {cnt[:, 0].tolist()} final detections")


def test_e2e_citypersons_8s_vs_reference(cuda):
    """citypersons/mscnn-8s-1344-2x at 2x3x192x384: eight heads, bbox normalisation in BoxOutput, Deconvolution 2x and
    8x4 ROI pooling at 1/4, DecodeBBox and Softmax on the one stage."""
    g = np.load(GOLD / "e2e_citypersons_8s_192x384.npz")
    n, h, w = 2, 192, 384
    net = _build(_deploy("citypersons/mscnn-8s-1344-2x", n, h, w), n, h, w)
    net.forward_only()
    _check_trunk_and_heads(net, g, ["conv4_3", "conv4_3_2x", "conv5_3", "conv6_1"], 8)
    out = {k: net.blob(k) for k in ("proposals_score", "cls_pred", "bbox_pred")}
    assert net.blob("roi_pool").shape[1:] == (1024, 8, 4)
    _check_rows_and_head(out, g, 1e-3, 0.997, 0.99, 0.98, "citypersons 8s 192x384")
    m = _match_rows(_stage_rows({k: net.blob(k) for k in ("output_bbox_1st", "cls_prob_1st")}, "1st", 1),
                    _stage_rows(g, "1st", 1), 1e-3)
    print(f"citypersons 8s: decoded boxes and probabilities matched {m:.4f}")
    assert m >= 0.95, m


def test_e2e_citypersons_cascade_vs_reference_and_detect_classes(cuda):
    """citypersons/cascade-mscnn-8s-1344-2x at 2x3x192x384, at the bars and KITTI floors of
    test_e2e_cascade_vs_reference; the Eltwise average checked as its wider branch does.  Then
    Net.detect_cascade_classes on cls_prob_3rd_avg with the CityPersons driver's settings against the restated
    run_cascademscnn.m post-process on the net's own outputs."""
    import detect_classes_ref as R
    from mscnn_b200 import drivers
    g = np.load(GOLD / "e2e_citypersons_cascade_192x384.npz")
    n, h, w = 2, 192, 384
    net = _build(_deploy("citypersons/cascade-mscnn-8s-1344-2x", n, h, w), n, h, w)
    net.forward_only()
    _check_trunk_and_heads(net, g, ["conv4_3", "conv4_3_2x", "conv5_3", "conv6_1"], 8)
    same_rows = net.blob("proposals").shape == g["proposals"].shape
    for b in ["roi_pool", "fc6"]:
        x = net.blob(b)
        if tuple(g[b + "__shape"]) != x.shape:
            assert not same_rows
            continue
        sub, ref, m2 = x.reshape(-1)[::SUB], g[b + "__sub"], float(g[b + "__m2"][0])
        frac = _rel_ok(sub, ref, 1e-3, m2).mean()
        assert frac >= 0.97, (b, frac)
    ref_ps, got_ps = g["proposals_score"].reshape(-1, 6), net.blob("proposals_score").reshape(-1, 6)
    assert abs(len(got_ps) - len(ref_ps)) <= max(3, len(ref_ps) // 100)
    assert _match_rows(got_ps, ref_ps, 1e-3) >= 0.97
    names = ["output_bbox_1st", "output_bbox_2nd", "output_bbox_3rd", "cls_prob_1st", "cls_prob_2nd", "cls_prob_3rd",
             "cls_prob_1st_3rd", "cls_prob_2nd_3rd", "cls_prob_3rd_avg"]
    blobs = {k: net.blob(k) for k in names}
    matched = {}
    for stage, floor in zip(["1st", "2nd", "3rd"], (0.95, 0.90, 0.85)):
        matched[stage] = _match_rows(_stage_rows(blobs, stage, 1), _stage_rows(g, stage, 1), 1e-3)
        assert matched[stage] >= floor, (stage, matched[stage])
    avg = dict(blobs, cls_prob_avg=blobs["cls_prob_3rd_avg"], output_bbox_avg=blobs["output_bbox_3rd"])
    gavg = {"cls_prob_avg": g["cls_prob_3rd_avg"], "output_bbox_avg": g["output_bbox_3rd"]}
    matched["3rd_avg"] = _match_rows(_stage_rows(avg, "avg", 1), _stage_rows(gavg, "avg", 1), 1e-3)
    print(f"citypersons cascade: proposals {len(got_ps)} vs {len(ref_ps)}, stage rows matched {matched}")
    assert matched["3rd_avg"] >= 0.85
    third = np.float32(0.33333333)
    manual = blobs["cls_prob_1st_3rd"] * third + blobs["cls_prob_2nd_3rd"] * third + blobs["cls_prob_3rd"] * third
    np.testing.assert_allclose(blobs["cls_prob_3rd_avg"], manual, rtol=1e-6)
    np.testing.assert_allclose(blobs["cls_prob_3rd_avg"].sum(1), 1.0, rtol=1e-5)

    cfg, classes = _cfg(drivers.CITYPERSONS, h, w, (384, 768))
    dets = torch.zeros((n, 1, cfg.max_rois_per_image, 5), device=cuda)
    cnt = torch.zeros((n, 1), dtype=torch.int32, device=cuda)
    net.detect_cascade_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr(), stage="3rd", cls_prob="cls_prob_3rd_avg")
    torch.cuda.synchronize()
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    props = net.blob("proposals_3rd").reshape(-1, 5)
    prob = blobs["cls_prob_3rd_avg"].reshape(len(props), -1)
    outb = blobs["output_bbox_3rd"].reshape(-1, 5)
    start = 0
    for i in range(n):
        sl = slice(start, start + net.num_proposals(i))
        ref, = R.cascade_detect_postprocess_classes(props[sl], prob[sl], outb[sl], [2], overlap=cfg.nms_overlap,
                                                    ratios=(cfg.ratio_h, cfg.ratio_w), org_hw=(cfg.org_h, cfg.org_w))
        assert cnt[i, 0] == len(ref), (i, cnt[i, 0], len(ref))
        np.testing.assert_allclose(dets[i, 0, :cnt[i, 0]], ref, rtol=1e-5, atol=1e-5)
        start = sl.stop
    assert start == len(props) and cnt.sum() > 0
    print(f"citypersons cascade: {cnt[:, 0].tolist()} final detections")


# ------------------------------------------------------------------------------------------------ stages isolated
def _ref_and_net(proto, n, h, w):
    """The reference net run live (oracle/_ref) and our net run to its end, both on the same synthetic weights and
    images."""
    from oracle import ref
    from mscnn_b200 import synth
    rnet = ref.RefNet(proto, is_path=False)
    layers = [(nm, t, rnet.param_shapes(nm)) for nm, t in zip(rnet.layer_names, rnet.layer_types)]
    rnet.set_params(synth.make_weights(layers))
    rnet.set_blob("data", synth.make_images(n, h, w))
    rnet.forward()
    net = _build(proto, n, h, w)
    net.forward_only()
    return rnet, net


def _inject(net, rnet, feat):
    """The reference's `feat` and proposals into every Split top of them that the detection stages read."""
    fmap, props = rnet.blob(feat), rnet.blob("proposals")
    hit = 0
    for b in net.blob_names:
        if b.startswith(feat + "_") and "_split_" in b and not b.startswith(feat + "_2x"):
            net.set_input(b, fmap)
            hit += 1
        if b.startswith("proposals_proposals_0_split_"):
            net.set_input(b, props)
            hit += 1
    assert hit >= 3, hit


def _row_errors(a, r, name):
    a, r = a.reshape(a.shape[0], -1), r.reshape(r.shape[0], -1)
    if name.startswith(("proposals", "output_bbox")):     # boxes: relative to the box extent
        ext = np.maximum(np.maximum(r[:, 3] - r[:, 1], r[:, 4] - r[:, 2]), 1.0)[:, None]
        err = np.abs(a - r) / ext
    else:
        m2 = float(np.mean(r.astype(np.float64) ** 2))
        err = np.abs(a - r) / (np.abs(r) + np.sqrt(m2))
    return err.max(axis=1)


def test_caltech_head_stage_isolated_vs_reference(cuda):
    """roi_pool_org through bbox_pred fed with the reference's conv4_3 and proposals: every row of roi_pool (8x4 bins of
    the org || ctx pair), roi_c1 (3x3 pad 1 on the 8x4 grid), fc6 (K = 16384), cls_pred and bbox_pred within 1e-3."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not present")
    n, h, w = 1, 144, 192
    rnet, net = _ref_and_net(_deploy("caltech/mscnn-7s-720", n, h, w), n, h, w)
    _inject(net, rnet, "conv4_3")
    net.forward_only(start="roi_pool_org")
    worst = {}
    for name in ("roi_pool", "roi_c1", "fc6", "cls_pred", "bbox_pred"):
        a, r = net.blob(name), rnet.blob(name)
        assert a.shape == r.shape, name
        worst[name] = float(_row_errors(a, r, name).max())
    print("caltech stages, worst error:", worst, "rows", rnet.blob("proposals").shape[0])
    assert rnet.blob("roi_pool").shape[1:] == (1024, 8, 4)
    for name, e in worst.items():
        assert e <= 1e-3, (name, e)


def test_citypersons_cascade_stages_isolated_vs_reference(cuda):
    """The three stages of the CityPersons cascade fed with the reference's conv4_3_2x and proposals, at the bars of
    test_cascade_stages_isolated_vs_reference's kitti branch (every row of the first stage within 1e-3; the later stages
    pool boxes that carry a 1e-5 error through round(), >= 98 % of rows); the Eltwise average and its two Softmax
    inputs are held to the same bars as the third stage they come from."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not present")
    n, h, w = 2, 128, 256
    rnet, net = _ref_and_net(_deploy("citypersons/cascade-mscnn-8s-1344-2x", n, h, w), n, h, w)
    _inject(net, rnet, "conv4_3_2x")
    net.forward_only(start="roi_pool_org")
    names = ["cls_pred", "bbox_pred", "proposals_2nd", "cls_pred_2nd", "bbox_pred_2nd", "proposals_3rd", "cls_pred_3rd",
             "bbox_pred_3rd", "output_bbox_1st", "output_bbox_2nd", "output_bbox_3rd", "cls_prob_1st", "cls_prob_2nd",
             "cls_prob_3rd", "cls_prob_1st_3rd", "cls_prob_2nd_3rd", "cls_prob_3rd_avg"]
    worst = {}
    for name in names:
        a, r = net.blob(name), rnet.blob(name)
        assert a.shape == r.shape, name
        err = _row_errors(a, r, name)
        ok_rows = float((err <= 1e-3).mean())
        worst[name] = (ok_rows, float(err.max()))
        if name in ("cls_pred", "bbox_pred", "proposals_2nd", "output_bbox_1st", "cls_prob_1st"):
            assert ok_rows == 1.0, (name, worst[name])
        else:
            assert ok_rows >= 0.98, (name, worst[name])
    print("citypersons cascade stages (rows within 1e-3, worst error):", worst, "rows", rnet.blob("proposals").shape[0])
