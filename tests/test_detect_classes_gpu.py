"""The several-class post-process on the device (mscnn_detect_postprocess_classes, the cascade and packed forms, the
Net-facade entries): N images x C classes run as N * C class slots through the single-class pipeline.

* every slot (n, c) equals, bit for bit, the single-class entry with cls_id = cls_ids[c] (MS-CNN and cascade, padded
  and packed, with and without per-image geometry, both class orders, N * C across a 64-slot launch chunk);
* det_thr > 0 equals the unthresholded result without its rows of prob < det_thr, bit for bit; det_thr <= 0 is off;
* the hand-derived vectors (tests/golden/a15_classes_cases.json);
* the KITTI pedestrian / cyclist net end to end against the reference's own layers (e2e_pedcyc_8s_192x640.npz) and
  Net.detect_classes against the restated per-class MATLAB loop on the net's own outputs;
* one two-class call launches fewer kernels than two single-class calls; the pushed payload equals detect_classes."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"
CASES = json.loads((GOLD / "a15_classes_cases.json").read_text())["cases"]
SUB = 7919


def _cfg(num_cls, cls_id=2, cap=1024, overlap=0.5):
    from mscnn_b200 import capi
    cfg = capi.DetectCfg()
    cfg.num_cls, cfg.cls_id = num_cls, cls_id
    for k, v in enumerate([0.1, 0.1, 0.2, 0.2]):
        cfg.bbox_std[k], cfg.bbox_mean[k] = v, 0.0
    cfg.proposal_thr, cfg.nms_overlap = -10.0, overlap
    cfg.ratio_h, cfg.ratio_w = 1.25, 0.8
    cfg.org_h, cfg.org_w = 768.0 / 1.25, 2560.0 / 0.8
    cfg.max_rois_per_image = cap
    return cfg


def _inputs(cuda, n, cascade, seed=5, num_cls=3):
    """Synthetic post-process inputs of n images (one of them empty when n > 1), ROIs dense enough for NMS to act."""
    rng = np.random.default_rng(seed + n)
    counts = [int(v) for v in rng.integers(40, 400, n)]
    if n > 1:
        counts[1] = 0
    r = sum(counts)
    img = np.repeat(np.arange(n), counts).astype(np.float32)
    x1, y1 = rng.uniform(0, 2400, r), rng.uniform(0, 700, r)
    w, h = rng.uniform(15, 300, r), rng.uniform(15, 200, r)
    num_out = np.array([max(r, 1), r] + counts, dtype=np.int32)
    if cascade:
        prop = np.stack([img, x1, y1, x1 + w, y1 + h], axis=1).astype(np.float32)
        prop[3, 3] = prop[3, 1] - 1                      # zero width under the "+ 1" convention: dropped
        z = rng.standard_normal((r, num_cls)) * 2
        cls = (np.exp(z) / np.exp(z).sum(1, keepdims=True)).astype(np.float32)
        jit = rng.normal(0, 8, (r, 4))
        bbox = np.concatenate([img[:, None], prop[:, 1:] + jit], axis=1).astype(np.float32)
    else:
        sc = rng.uniform(-12, 10, r)
        prop = np.stack([img, x1, y1, x1 + w, y1 + h, sc], axis=1).astype(np.float32)
        prop[5, 3] = prop[5, 1]                          # zero width: dropped
        cls = (rng.standard_normal((r, num_cls)) * 2).astype(np.float32)
        bbox = rng.standard_normal((r, 4 * num_cls)).astype(np.float32)
    if r > 7:
        cls[7, 1] = np.nan                               # NaN row: dropped in every class
    dev = [torch.from_numpy(a).to(cuda) for a in (prop, cls, bbox, num_out)]
    return (prop, cls, bbox, counts), dev


def _geometry(n, on):
    if not on:
        return None
    rng = np.random.default_rng(n)
    g = np.zeros((n, 4), np.float32)
    g[:, 0], g[:, 1] = rng.uniform(0.5, 2.0, n), rng.uniform(0.5, 2.0, n)
    g[:, 2], g[:, 3] = 768.0 / g[:, 0], 2560.0 / g[:, 1]
    return g


def _bits(t):
    return t.cpu().numpy().view(np.int32)


def _single(cfg, cascade, n, dev, cls_id, geom):
    from mscnn_b200 import ops
    cfg.cls_id = cls_id
    f = ops.cascade_detect_postprocess if cascade else ops.detect_postprocess
    return f(cfg, n, *dev, geometry=geom)


@pytest.mark.parametrize("geom_on", [False, True], ids=["cfg_geometry", "per_image_geometry"])
@pytest.mark.parametrize("cls_ids", [[2, 3], [3, 2]], ids=["ids_2_3", "ids_3_2"])
@pytest.mark.parametrize("n", [1, 3, 33])
@pytest.mark.parametrize("cascade", [False, True], ids=["mscnn", "cascade"])
def test_every_slot_equals_the_single_class_call_bit_for_bit(cuda, cascade, n, cls_ids, geom_on):
    from mscnn_b200 import capi, ops, parallel
    cfg = _cfg(3)
    k = capi.DetectClasses.of(cls_ids)
    _, dev = _inputs(cuda, n, cascade)
    geom = _geometry(n, geom_on)
    f = ops.cascade_detect_postprocess_classes if cascade else ops.detect_postprocess_classes
    dets, cnt = f(cfg, k, n, *dev, geometry=geom)
    packed = None if cascade else ops.detect_postprocess_classes_packed(cfg, k, n, *dev, geometry=geom)
    torch.cuda.synchronize()
    assert tuple(dets.shape) == (n, len(cls_ids), cfg.max_rois_per_image, 5) and tuple(cnt.shape) == (n, len(cls_ids))
    slots = parallel.unpack_payload(packed, 1, n * len(cls_ids), cfg.max_rois_per_image) if packed is not None else None
    total = 0
    for c, cid in enumerate(cls_ids):
        d1, c1 = _single(cfg, cascade, n, dev, cid, geom)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(cnt[:, c].contiguous()), _bits(c1)), (c, cid)
        assert np.array_equal(_bits(dets[:, c].contiguous()), _bits(d1)), (c, cid)
        c1 = c1.cpu().numpy()
        d1 = d1.cpu().numpy()
        total += int(c1.sum())
        if slots is not None:
            for i in range(n):
                got = slots[i * len(cls_ids) + c]
                assert np.array_equal(got.view(np.int32), d1[i, :c1[i]].view(np.int32)), (i, c)
    assert total > 0


@pytest.mark.parametrize("cascade", [False, True], ids=["mscnn", "cascade"])
def test_det_thr_equals_the_unthresholded_result_without_low_rows(cuda, cascade):
    """det_thr = 0.05: each slot = the det_thr-off slot minus its rows of prob < 0.05 (fp32), bit for bit, and some rows
    do go; det_thr = 0 and -1 leave the result unchanged."""
    from mscnn_b200 import capi, ops
    cfg = _cfg(3)
    n, ids = 3, [2, 3]
    _, dev = _inputs(cuda, n, cascade, seed=11)
    f = ops.cascade_detect_postprocess_classes if cascade else ops.detect_postprocess_classes
    d_off, c_off = (t.cpu().numpy() for t in f(cfg, capi.DetectClasses.of(ids, -1.0), n, *dev))
    d_thr, c_thr = (t.cpu().numpy() for t in f(cfg, capi.DetectClasses.of(ids, 0.05), n, *dev))
    dropped = 0
    for i in range(n):
        for c in range(len(ids)):
            full = d_off[i, c, :c_off[i, c]]
            want = full[full[:, 4] >= np.float32(0.05)]
            dropped += len(full) - len(want)
            assert c_thr[i, c] == len(want), (i, c)
            assert np.array_equal(d_thr[i, c, :c_thr[i, c]].view(np.int32), want.view(np.int32)), (i, c)
    assert dropped > 0
    for off in (0.0, -1.0):
        d, c = (t.cpu().numpy() for t in f(cfg, capi.DetectClasses.of(ids, off), n, *dev))
        assert np.array_equal(c, c_off) and np.array_equal(d.view(np.int32), d_off.view(np.int32)), off


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_classes_hand_vectors_device(cuda, case):
    from mscnn_b200 import capi, ops
    cascade = case["kind"] == "cascade_classes"
    cfg = _cfg(case["num_cls"], cap=64)
    cfg.ratio_h, cfg.ratio_w = case["ratios"]
    cfg.org_h, cfg.org_w = case.get("org_hw", case["net_hw"])
    k = capi.DetectClasses.of(case["cls_ids"], case["det_thr"])
    names = ("proposals", "cls_prob", "output_bbox") if cascade else ("proposals_score", "cls_pred", "bbox_pred")
    arrs = [torch.from_numpy(np.array(case[nm], np.float32)).to(cuda) for nm in names]
    r = arrs[0].shape[0]
    num_out = torch.tensor([r, r, r], dtype=torch.int32, device=cuda)
    f = ops.cascade_detect_postprocess_classes if cascade else ops.detect_postprocess_classes
    dets, cnt = f(cfg, k, 1, *arrs, num_out)
    torch.cuda.synchronize()
    for c, want in enumerate(case["dets"]):
        got = dets[0, c, :int(cnt[0, c].item())].cpu().numpy()
        want = np.array(want, dtype=np.float64).reshape(-1, 5)
        assert got.shape == want.shape, (c, got, case["derivation"])
        np.testing.assert_allclose(got, want, rtol=case["tol"], atol=case["tol"], err_msg=case["derivation"])


def _pedcyc_deploy(n, h, w):
    """The shipped kitti_ped_cyc/mscnn-8s-768-trainval deploy file with its input set to n x 3 x h x w."""
    import re
    import tarfile
    with tarfile.open(GOLD / "deploy.tar.xz") as t:
        text = t.extractfile("deploy/kitti_ped_cyc/mscnn-8s-768-trainval/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: 768\s+input_dim: 2560",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def _pedcyc_net(n, h, w):
    from mscnn_b200 import net as mnet, synth
    mnet.set_precision("fp32")
    net = mnet.Net(_pedcyc_deploy(n, h, w))
    net.set_params(synth.make_weights(net.layers()))
    return net


def test_e2e_pedcyc_8s_vs_reference_and_detect_classes(cuda):
    """The pedestrian / cyclist net (eight 7-channel heads, cls_pred 3, bbox_pred 12) at 2x3x192x640 against the
    reference's own layers, to the bounds of test_net_gpu.py::test_e2e_kitti_8s_vs_reference; then
    Net.detect_classes([2, 3]) against the driver's per-class loop (kitti_ped_cyc/run_mscnn_detection.m:93-121) on the
    net's own outputs, to the tolerance of test_net_gpu.py::test_final_detections_vs_oracle."""
    import detect_classes_ref as R
    from mscnn_b200 import net as mnet, synth
    from test_net_gpu import _check_rows_and_head, _rel_ok
    g = np.load(GOLD / "e2e_pedcyc_8s_192x640.npz")
    n, h, w = 2, 192, 640
    net = _pedcyc_net(n, h, w)
    out = net.forward(data=synth.make_images(n, h, w))
    for b in ["conv4_3", "conv5_3", "conv6_1"]:
        x = net.blob(b)
        assert tuple(g[b + "__shape"]) == x.shape
        sub, ref, m2 = x.reshape(-1)[::SUB], g[b + "__sub"], float(g[b + "__m2"][0])
        assert _rel_ok(sub, ref, 1e-3, m2).mean() >= 0.999, b
    heads = [k for k in g.files if k.startswith("LFCN_")]
    assert len(heads) == 8
    for b in heads:
        x, ref = net.blob(b), g[b]
        assert x.shape[1] == 7
        m2 = float(np.mean(ref.astype(np.float64) ** 2))
        assert _rel_ok(x, ref, 1e-3, m2).mean() >= 0.999, b
    assert out["cls_pred"].shape[1] == 3 and out["bbox_pred"].shape[1] == 12
    _check_rows_and_head(out, g, 1e-3, 0.997, 0.99, 0.98, "pedcyc 8s 192x640")

    cfg, k = mnet.kitti_ped_cyc_detect_cfg(h, w)
    dets = torch.zeros((n, 2, cfg.max_rois_per_image, 5), device=cuda)
    cnt = torch.zeros((n, 2), dtype=torch.int32, device=cuda)
    net.detect_classes(cfg, k, dets.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    ps = out["proposals_score"].reshape(-1, 6)
    start = 0
    for i in range(n):
        sl = slice(start, start + net.num_proposals(i))
        refs = R.detect_postprocess_classes(ps[sl], out["cls_pred"][sl], out["bbox_pred"][sl], [2, 3], net_hw=(h, w))
        for c, ref in enumerate(refs):
            assert cnt[i, c] == len(ref), (i, c)
            np.testing.assert_allclose(dets[i, c, :cnt[i, c]], ref, rtol=1e-5, atol=1e-5)
        start = sl.stop
    assert cnt.sum() > 0


def test_two_class_call_launches_fewer_kernels_and_push_equals_detect_classes(cuda):
    """mscnn_kernel_launch_count of one two-class call < two single-class calls; the single-rank push of the two-class
    payload (an exchange sized for batch x 2 slots) equals detect_classes, over consecutive steps (both generations),
    following test_multigpu_gpu.py::test_detect_push_single_rank_equals_detect; an exchange sized for the batch alone
    is refused."""
    from mscnn_b200 import capi, net as mnet, parallel, synth
    mnet.set_stream(torch.cuda.current_stream().cuda_stream)
    b, h, w = 3, 192, 640
    net = _pedcyc_net(b, h, w)
    cfg, k = mnet.kitti_ped_cyc_detect_cfg(h, w)
    cap = cfg.max_rois_per_image
    L = capi.lib()
    x = parallel.PeerExchange(b * 2, cap, rank=0, world=1, generations=2)
    x_small = parallel.PeerExchange(b, cap, rank=0, world=1, generations=2)
    try:
        for step in range(3):
            net.forward(data=synth.make_images(b, h, w, first_index=step * b))
            dets = torch.zeros((b, 2, cap, 5), device=cuda)
            cnt = torch.zeros((b, 2), dtype=torch.int32, device=cuda)
            n0 = L.mscnn_kernel_launch_count()
            net.detect_classes(cfg, k, dets.data_ptr(), cnt.data_ptr())
            n1 = L.mscnn_kernel_launch_count()
            one = torch.zeros((b, cap, 5), device=cuda)
            one_cnt = torch.zeros(b, dtype=torch.int32, device=cuda)
            for cid in (2, 3):
                cfg.cls_id = cid
                net.detect(cfg, one.data_ptr(), one_cnt.data_ptr())
            n2 = L.mscnn_kernel_launch_count()
            assert 0 < n1 - n0 < n2 - n1, (n1 - n0, n2 - n1)
            net.detect_push_classes(cfg, k, x)
            x.wait(torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            got = parallel.unpack_payload(x.gathered(), 1, b * 2, cap)
            d, c = dets.cpu().numpy(), cnt.cpu().numpy()
            assert int(c.sum()) > 0
            for i in range(b):
                for s in range(2):
                    assert np.array_equal(got[i * 2 + s], d[i, s, :c[i, s]]), (step, i, s)
        with pytest.raises(capi.MscnnError):
            net.detect_push_classes(cfg, k, x_small)
    finally:
        x.close()
        x_small.close()
