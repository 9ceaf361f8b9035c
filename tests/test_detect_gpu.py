"""GPU parity of the HBM / latency-bound stages against the CPU oracle (oracle.port, itself
pinned to the verbatim reference build in tests/test_oracle.py):
BoxOutput (decode + top-N + NMS), ROIPooling(+pad_ratio, fused concat), Pooling, depthwise
Deconvolution 2x, and the final-detection post-process.  All calls go through the C ABI.

Bar: integer / index / ordering results bit-exact; box coordinates within 2 ulp (the device
evaluates exp() in fp64 and rounds once, the reference calls expf); plane kernels exact when
inputs are bf16-representable."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import port

pytestmark = pytest.mark.gpu

FIELDS_A = dict(field_w=[60, 84, 120, 168, 240, 336, 480, 672], field_h=[60, 84, 120, 168, 240, 336, 480, 672],
                rate=[8, 8, 16, 16, 32, 32, 64, 64])


def _maps(rng, n, ch, shapes, score_scale=3.0, box_scale=0.4, quant=None, bg_bias=0.0):
    maps = []
    for (h, w) in shapes:
        m = rng.standard_normal((n, ch, h, w)).astype(np.float32)
        m[:, : ch - 4] *= score_scale
        m[:, ch - 4:] *= box_scale
        m[:, 0] += bg_bias
        if quant:
            m[:, : ch - 4] = np.round(m[:, : ch - 4] / quant) * quant   # many exact score ties
        maps.append(m)
    return maps


def _run_gpu(cuda, maps, **kw):
    from mscnn_b200 import ops
    shapes = [(m.shape[1], m.shape[2], m.shape[3]) for m in maps]
    cfg = ops.make_box_cfg(shapes, kw["field_w"], kw["field_h"], kw["rate"], kw.get("fg_thr", 0.0),
                           kw.get("iou_thr", 0.5), kw.get("nms_type", "IOU"), kw.get("field_whr", 2.0),
                           kw.get("field_xyr", 2.0), kw.get("min_size", 15.0), kw["max_nms_num"],
                           kw.get("max_post_nms_num", 0), kw.get("bbox_mean"), kw.get("bbox_std"))
    dm = [torch.from_numpy(m).to(cuda) for m in maps]
    rois, rois_score, num_out = ops.box_output_forward(cfg, dm)
    torch.cuda.synchronize()
    no = num_out.cpu().numpy()
    rows = int(no[0])
    return rois[:rows].cpu().numpy(), rois_score[:rows].cpu().numpy(), no


def _run_cpu(maps, **kw):
    return port.box_output(maps, kw["field_w"], kw["field_h"], kw["rate"], kw.get("fg_thr", 0.0),
                           kw.get("iou_thr", 0.5), kw.get("nms_type", "IOU"), kw.get("field_whr", 2.0),
                           kw.get("field_xyr", 2.0), kw.get("min_size", 15.0), kw["max_nms_num"],
                           kw.get("max_post_nms_num", 0), kw.get("bbox_mean"), kw.get("bbox_std"))


def _compare_boxes(g, c):
    g_rois, g_sc, g_no = g
    c_rois, c_sc, c_per, c_true = c
    assert g_no[1] == c_true, f"proposal count {g_no[1]} vs oracle {c_true}"
    assert list(g_no[2:]) == list(c_per), f"per-image counts {list(g_no[2:])} vs {list(c_per)}"
    assert g_rois.shape == c_rois.shape
    assert np.array_equal(g_rois[:, 0], c_rois[:, 0])
    assert np.array_equal(g_sc[:, 5], c_sc[:, 5]), "scores (and hence ranking) must be bit-exact"
    np.testing.assert_allclose(g_rois, c_rois, rtol=3e-7, atol=0)
    np.testing.assert_allclose(g_sc, c_sc, rtol=3e-7, atol=0)
    return float(np.mean(g_rois == c_rois))


SHAPES_A_SMALL = [(24, 80), (24, 80), (12, 40), (12, 40), (6, 20), (6, 20), (3, 10), (3, 10)]


@pytest.mark.parametrize("case", ["kitti_like", "ties", "cap_not_hit", "iomu", "post_cap"])
def test_box_output_parity(cuda, case):
    rng = np.random.default_rng(1706)
    kw = dict(FIELDS_A, fg_thr=-5.0, iou_thr=0.65, max_nms_num=300)
    quant = None
    n = 2
    if case == "ties":
        quant = 1.0
    if case == "cap_not_hit":
        kw["fg_thr"] = 6.0
    if case == "iomu":
        kw["nms_type"] = "IOMU"
    if case == "post_cap":
        kw["max_post_nms_num"] = 50
    maps = _maps(rng, n, 9, SHAPES_A_SMALL, quant=quant)
    frac = _compare_boxes(_run_gpu(cuda, maps, **kw), _run_cpu(maps, **kw))
    assert frac > 0.99   # at most a handful of 1-ulp coordinate differences


def test_box_output_full_size_config_a(cuda):
    """mscnn-8s-768 geometry: 81,600 anchors / image, top-2000, batch 2."""
    rng = np.random.default_rng(7)
    shapes = [(96, 320), (96, 320), (48, 160), (48, 160), (24, 80), (24, 80), (12, 40), (12, 40)]
    kw = dict(FIELDS_A, fg_thr=-5.0, iou_thr=0.65, max_nms_num=2000)
    maps = _maps(rng, 2, 9, shapes, bg_bias=2.0)
    g = _run_gpu(cuda, maps, **kw)
    _compare_boxes(g, _run_cpu(maps, **kw))
    assert g[2][1] > 500


def test_box_output_wider_config(cuda):
    """WIDER mscnn-12s-2x: 12 bottoms x 6 channels, bbox de-normalisation, fg_thr -3, whr 4, xyr 1,
    min_size 5, top-3000 (examples/widerface/mscnn-12s-2x/mscnn_deploy.prototxt:753-801)."""
    rng = np.random.default_rng(11)
    rates = [4] * 5 + [8] * 2 + [16] * 2 + [32] * 3
    fields = [12, 16, 24, 32, 48, 64, 96, 128, 192, 256, 384, 480]
    shapes = [(192 // r * 1, 256 // r * 1) for r in rates]
    kw = dict(field_w=fields, field_h=fields, rate=rates, fg_thr=-3.0, iou_thr=0.65, field_whr=4.0,
              field_xyr=1.0, min_size=5.0, max_nms_num=3000, bbox_mean=[0, 0, 0, 0], bbox_std=[0.1, 0.1, 0.2, 0.2])
    maps = _maps(rng, 2, 6, shapes, box_scale=4.0)
    _compare_boxes(_run_gpu(cuda, maps, **kw), _run_cpu(maps, **kw))


def test_box_output_empty_and_partial(cuda):
    """No candidate at all -> dummy ROI [0 1 1 10 10] and a zero score row
    (box_output_layer.cpp:195-199,214-218); one empty image inside a batch is skipped (:166)."""
    rng = np.random.default_rng(3)
    kw = dict(FIELDS_A, fg_thr=100.0, iou_thr=0.65, max_nms_num=300)
    maps = _maps(rng, 2, 9, SHAPES_A_SMALL)
    g_rois, g_sc, g_no = _run_gpu(cuda, maps, **kw)
    assert list(g_no[:2]) == [1, 0]
    assert g_rois.tolist() == [[0.0, 1.0, 1.0, 10.0, 10.0]] and not g_sc.any()
    c = _run_cpu(maps, **kw)
    assert c[3] == 0 and c[0].tolist() == g_rois.tolist()
    kw["fg_thr"] = -5.0
    for m in maps:
        m[0, 0] += 1000.0   # image 0: background wins everywhere
    _compare_boxes(_run_gpu(cuda, maps, **kw), _run_cpu(maps, **kw))


def _bf16_exact(a):
    return torch.from_numpy(a).bfloat16().float().numpy()


ROI_POOL_CASES = [(pr, s, p, c) for c in (128, 512) for pr, s, p in [(0.0, 0.125, 7), (0.25, 0.125, 7), (0.25, 0.25, 5)]]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
# C = 512 (conv4_3): every lane pools two channel groups.  The C = 128 cases keep their original ids.
@pytest.mark.parametrize("pad_ratio,scale,pooled,c", ROI_POOL_CASES,
                         ids=[f"{pr}-{s}-{p}" + ("" if c == 128 else f"-c{c}") for pr, s, p, c in ROI_POOL_CASES])
def test_roi_pool_parity(cuda, split, pad_ratio, scale, pooled, c):
    from mscnn_b200 import ops
    rng = np.random.default_rng(5)
    n, h, w = 2, 24, 80
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    img_w, img_h = w / scale, h / scale
    r = 200
    x1 = rng.uniform(-20, img_w, r); y1 = rng.uniform(-20, img_h, r)
    bw = rng.uniform(1, 300, r); bh = rng.uniform(1, 200, r)
    rois = np.stack([rng.integers(0, n, r), x1, y1, x1 + bw, y1 + bh], axis=1).astype(np.float32)
    rois[0] = [0, 1, 1, 10, 10]                   # the dummy ROI
    rois[1] = [1, 50, 40, 30, 20]                 # malformed: x2 < x1 -> forced 1x1 (:80-81)
    rois[2] = [0, img_w + 100, img_h + 100, img_w + 200, img_h + 200]   # outside -> empty bins -> 0
    rois[3] = [1, 3.5, 4.5, 4.5, 5.5]             # half-pixel coordinates: round() away from zero
    ref = port.roi_pool(x, rois, pooled, pooled, scale, pad_ratio)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    out = ops.roi_pool_forward(xp, torch.from_numpy(rois).to(cuda), r, pooled, scale, pad_ratio)
    got = ops.planes_to_nchw(out).cpu().numpy()
    assert np.array_equal(got, ref)


def test_roi_pool_fused_concat(cuda):
    """org || ctx written into one [R,7,7,2C] tensor == ConcatLayer of the two ROIPooling tops."""
    from mscnn_b200 import ops
    rng = np.random.default_rng(9)
    n, c, h, w = 1, 64, 12, 40
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    rois = np.array([[0, 8, 8, 100, 60], [0, 120, 10, 300, 90], [0, 0, 0, 319, 95]], dtype=np.float32)
    ref = port.concat_channels(port.roi_pool(x, rois, 7, 7, 0.125, 0.0), port.roi_pool(x, rois, 7, 7, 0.125, 0.25))
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), True)
    dr = torch.from_numpy(rois).to(cuda)
    out = ops.roi_pool_forward(xp, dr, 3, 7, 0.125, 0.0, out_channels=2 * c)
    out = ops.roi_pool_forward(xp, dr, 3, 7, 0.125, 0.25, out=out, channel_offset=c, out_channels=2 * c)
    got = ops.planes_to_nchw(out).cpu().numpy()
    assert np.array_equal(got, ref)


POOL_CASES = [("MAX", 24, 80, 2, 2), ("MAX", 9, 15, 2, 2), ("AVE", 12, 16, 2, 2), ("AVE", 7, 5, 2, 2),
              # stride 1 (the cascade nets' AVE 2/1 on the ROIAlign grid) and 3/2 windows that overlap, odd sizes
              ("MAX", 7, 9, 2, 1), ("AVE", 6, 11, 2, 1), ("MAX", 9, 15, 3, 2), ("AVE", 8, 13, 3, 2)]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("mode,h,w,k,s", POOL_CASES,
                         ids=[f"{m}-{h}-{w}" + ("" if (k, s) == (2, 2) else f"-k{k}s{s}") for m, h, w, k, s in POOL_CASES])
def test_pool_parity(cuda, split, mode, h, w, k, s):
    """2x2 stride 2, 2x2 stride 1 and 3x3 stride 2, including odd sizes where ceil mode adds a clipped last window
    (pooling_layer.cpp:90-93)."""
    from mscnn_b200 import capi, ops
    rng = np.random.default_rng(13)
    x = _bf16_exact(rng.standard_normal((2, 64, h, w)).astype(np.float32))
    ref = port.pool(x, k, s, 0, mode)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    out = ops.pool_forward(xp, k, s, capi.POOL_MAX if mode == "MAX" else capi.POOL_AVE)
    got = ops.planes_to_nchw(out).cpu().numpy()
    assert got.shape == ref.shape
    if mode == "MAX":
        assert np.array_equal(got, ref)
    else:
        np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_deconv2x_parity(cuda, split):
    """conv4_3_2x: depthwise 4x4 / stride 2 / pad 1 transposed conv with the bilinear filler."""
    from mscnn_b200 import ops, synth
    rng = np.random.default_rng(17)
    n, c, h, w = 2, 64, 9, 15
    x = _bf16_exact(np.abs(rng.standard_normal((n, c, h, w))).astype(np.float32))
    wt = np.broadcast_to(synth.bilinear_kernel(4), (c, 1, 4, 4)).astype(np.float32).copy()
    wt *= rng.uniform(0.5, 1.5, (c, 1, 1, 1)).astype(np.float32)    # not only the filler values
    ref = port.deconv_depthwise(x, wt, 2, 1)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    out = ops.deconv2x_forward(xp, torch.from_numpy(wt).to(cuda))
    got = ops.planes_to_nchw(out).cpu().numpy()
    assert got.shape == ref.shape == (n, c, 2 * h, 2 * w)
    np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)


def test_detect_postprocess_parity(cuda):
    """Final detections for the car class vs the restated MATLAB post-process."""
    from mscnn_b200 import capi, ops
    rng = np.random.default_rng(19)
    n = 3
    counts = [700, 0, 450]
    rows = []
    for i, cnt in enumerate(counts):
        x1 = rng.uniform(0, 2400, cnt); y1 = rng.uniform(0, 700, cnt)
        w = rng.uniform(15, 400, cnt); h = rng.uniform(15, 300, cnt)
        sc = rng.uniform(-12, 10, cnt)
        rows.append(np.stack([np.full(cnt, i), x1, y1, x1 + w, y1 + h, sc], axis=1))
    prop = np.concatenate(rows).astype(np.float32)
    prop[5, 3] = prop[5, 1]   # zero width -> dropped (run_mscnn_detection.m:82)
    r = len(prop)
    cls = (rng.standard_normal((r, 5)) * 2).astype(np.float32)
    bbox = rng.standard_normal((r, 20)).astype(np.float32)
    num_out = np.array([r, r] + counts, dtype=np.int32)
    cfg = capi.DetectCfg()
    cfg.num_cls, cfg.cls_id = 5, 2
    for k, v in enumerate([0.1, 0.1, 0.2, 0.2]):
        cfg.bbox_std[k] = v
        cfg.bbox_mean[k] = 0.0
    cfg.proposal_thr, cfg.nms_overlap = -10.0, 0.5
    cfg.ratio_h = cfg.ratio_w = 1.0
    cfg.org_h, cfg.org_w = 768.0, 2560.0
    cfg.max_rois_per_image = 2000
    dets, dcnt = ops.detect_postprocess(cfg, n, torch.from_numpy(prop).to(cuda), torch.from_numpy(cls).to(cuda),
                                        torch.from_numpy(bbox).to(cuda), torch.from_numpy(num_out).to(cuda))
    torch.cuda.synchronize()
    dets, dcnt = dets.cpu().numpy(), dcnt.cpu().numpy()
    start = 0
    for i, cnt in enumerate(counts):
        sl = slice(start, start + cnt)
        ref = port.detect_postprocess(prop[sl], cls[sl], bbox[sl], cls_id=2, net_hw=(768, 2560))
        assert dcnt[i] == len(ref), f"image {i}: {dcnt[i]} detections vs oracle {len(ref)}"
        np.testing.assert_allclose(dets[i, : dcnt[i]], ref, rtol=1e-6, atol=1e-6)
        start += cnt


# ------------------------------------------------------------------- cascade-net layers
@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("pad_ratio,scale,pooled", [(0.0, 0.125, 5), (0.25, 0.125, 5), (0.25, 0.25, 7)])
def test_roi_align_parity(cuda, split, pad_ratio, scale, pooled):
    """ROIAlign grid samples vs the restated roi_align_layer.cpp:49-139.  The inputs are bf16-exact, the
    interpolation is fp32 in the reference's order; the only difference is the storage of the result
    as bf16 planes (hi + lo: 2^-17 relative, hi only: 2^-9)."""
    from mscnn_b200 import ops
    rng = np.random.default_rng(23)
    n, c, h, w = 2, 128, 24, 40
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    img_w, img_h = w / scale, h / scale
    r = 150
    x1 = rng.uniform(-30, img_w, r); y1 = rng.uniform(-30, img_h, r)
    bw = rng.uniform(1, 200, r); bh = rng.uniform(1, 150, r)
    rois = np.stack([rng.integers(0, n, r), x1, y1, x1 + bw, y1 + bh], axis=1).astype(np.float32)
    rois[0] = [0, 1, 1, 10, 10]
    rois[1] = [1, 50, 40, 30, 20]                                        # malformed -> zeros (:94-97)
    rois[2] = [0, img_w + 100, img_h + 100, img_w + 200, img_h + 200]    # outside -> zeros (:104-108)
    rois[3] = [1, 3.5, 4.5, 4.5, 5.5]
    rois[4] = [0, 0, 0, img_w - 1, img_h - 1]
    ref = port.roi_align(x, rois, pooled, pooled, scale, pad_ratio)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    out = ops.roi_align_forward(xp, torch.from_numpy(rois).to(cuda), r, pooled, scale, pad_ratio)
    got = ops.planes_to_nchw(out).cpu().numpy()
    assert got.shape == ref.shape == (r, c, pooled + 1, pooled + 1)
    assert not got[1].any() and not got[2].any()
    np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)
    assert np.array_equal(got == 0, ref == 0)


def test_decode_bbox_parity(cuda):
    """DecodeBBox vs the restated decode_bbox_layer.cpp:53-124 / math_functions.cpp:46-77 and the golden
    vectors from the verbatim reference build: bit-exact up to expf's own last-bit error."""
    from mscnn_b200 import ops
    g = np.load(Path(__file__).resolve().parent / "golden" / "layers_cascade.npz")
    std = (0.05, 0.05, 0.1, 0.1)
    got = ops.decode_bbox_forward(torch.from_numpy(g["dec_b"]).to(cuda), torch.from_numpy(g["dec_p"]).to(cuda),
                                  (0, 0, 0, 0), std).cpu().numpy()
    assert np.array_equal(got, g["dec_out"].reshape(-1, 5))
    got = ops.decode_bbox_forward(torch.from_numpy(g["dec_b"]).to(cuda), torch.from_numpy(g["dec_p"]).to(cuda)).cpu().numpy()
    assert np.array_equal(got, g["dec_out_nostat"].reshape(-1, 5))
    rng = np.random.default_rng(29)
    r = 5000
    x1 = rng.uniform(-50, 2500, r); y1 = rng.uniform(-50, 700, r)
    prior = np.stack([rng.integers(0, 8, r), x1, y1, x1 + rng.uniform(-10, 500, r), y1 + rng.uniform(-10, 400, r)], 1).astype(np.float32)
    bbox = (rng.standard_normal((r, 8)) * 3).astype(np.float32)
    ref = port.decode_bbox(bbox, prior, (0.01, -0.02, 0.0, 0.03), (0.1, 0.1, 0.2, 0.2))
    got = ops.decode_bbox_forward(torch.from_numpy(bbox).to(cuda), torch.from_numpy(prior).to(cuda),
                                  (0.01, -0.02, 0.0, 0.03), (0.1, 0.1, 0.2, 0.2)).cpu().numpy()
    # glibc's expf differs from the correctly rounded exp by 1 ulp on ~0.06 % of its arguments (measured);
    # the device rounds the fp64 exp once.  Every other operation is the same IEEE fp32 op in the same order.
    bad_rows = (got != ref).any(axis=1)
    assert bad_rows.mean() <= 0.005, bad_rows.mean()
    ext = np.maximum(np.abs(ref[:, 1:]).max(axis=1, keepdims=True), 1.0)
    assert (np.abs(got[:, 1:] - ref[:, 1:]) <= 4e-7 * ext).all()


def test_softmax_eltwise_parity(cuda):
    from mscnn_b200 import capi, ops
    g = np.load(Path(__file__).resolve().parent / "golden" / "layers_cascade.npz")
    sm = ops.softmax_forward(torch.from_numpy(g["sm_x"]).to(cuda)).cpu().numpy()
    np.testing.assert_allclose(sm, g["sm_y"].reshape(6, 5), rtol=1e-6, atol=1e-12)
    rng = np.random.default_rng(31)
    x = (rng.standard_normal((300, 5, 3, 2)) * 4).astype(np.float32)
    for axis in (1, 3):
        got = ops.softmax_forward(torch.from_numpy(x).to(cuda), axis).cpu().numpy()
        assert np.array_equal(got, port.softmax(x, axis))          # same exp, same summation order
    a, b, c = (rng.standard_normal((1000, 5)).astype(np.float32) for _ in range(3))
    da, db, dc = (torch.from_numpy(v).to(cuda) for v in (a, b, c))
    cf = [0.33333333, -2.0, 0.5]
    assert np.array_equal(ops.eltwise_forward([da, db, dc], capi.ELTWISE_SUM, cf).cpu().numpy(), port.eltwise([a, b, c], "SUM", cf))
    assert np.array_equal(ops.eltwise_forward([da, db, dc], capi.ELTWISE_SUM).cpu().numpy(), port.eltwise([a, b, c], "SUM"))
    assert np.array_equal(ops.eltwise_forward([da, db, dc], capi.ELTWISE_PROD).cpu().numpy(), port.eltwise([a, b, c], "PROD"))
    assert np.array_equal(ops.eltwise_forward([da, db], capi.ELTWISE_MAX).cpu().numpy(), port.eltwise([a, b], "MAX"))
    assert np.array_equal(ops.eltwise_forward([da, db, dc], capi.ELTWISE_MAX).cpu().numpy(), port.eltwise([a, b, c], "MAX"))
    np.testing.assert_allclose(ops.eltwise_forward([torch.from_numpy(g["sm_x"]).to(cuda), torch.from_numpy(sm).to(cuda),
                                                    torch.from_numpy(g["sm_x"]).to(cuda)], capi.ELTWISE_SUM, cf).cpu().numpy(),
                               g["elt_sum"].reshape(6, 5), rtol=1e-6, atol=1e-6)


def test_cascade_detect_postprocess_parity(cuda):
    """Cascade final detections (run_cascademscnn.m:99-126) vs the restated MATLAB post-process."""
    from mscnn_b200 import capi, ops
    rng = np.random.default_rng(37)
    n = 3
    counts = [600, 0, 380]
    props, outs = [], []
    for i, cnt in enumerate(counts):
        x1 = rng.uniform(0, 1800, cnt); y1 = rng.uniform(0, 500, cnt)
        w = rng.uniform(15, 300, cnt); h = rng.uniform(15, 200, cnt)
        p = np.stack([np.full(cnt, i), x1, y1, x1 + w, y1 + h], axis=1)
        props.append(p)
        o = p.copy()
        o[:, 1:] += rng.normal(0, 6, (cnt, 4))
        outs.append(o)
    prop = np.concatenate(props).astype(np.float32)
    out = np.concatenate(outs).astype(np.float32)
    prop[7, 3] = prop[7, 1] - 1            # zero width in the "+1" convention -> dropped (:117)
    out[9, 1:] = [-40, -10, 2100, 700]     # clipped on all four sides
    r = len(prop)
    prob = port.softmax((rng.standard_normal((r, 5)) * 2).astype(np.float32))
    num_out = np.array([r, r] + counts, dtype=np.int32)
    cfg = capi.DetectCfg()
    cfg.num_cls, cfg.cls_id = 5, 2
    cfg.nms_overlap = 0.5
    cfg.ratio_h, cfg.ratio_w = 576.0 / 375.0, 1920.0 / 1242.0
    cfg.org_h, cfg.org_w = 375.0, 1242.0
    cfg.max_rois_per_image = 2000
    dets, dcnt = ops.cascade_detect_postprocess(cfg, n, torch.from_numpy(prop).to(cuda), torch.from_numpy(prob).to(cuda),
                                                torch.from_numpy(out).to(cuda), torch.from_numpy(num_out).to(cuda))
    torch.cuda.synchronize()
    dets, dcnt = dets.cpu().numpy(), dcnt.cpu().numpy()
    start = 0
    for i, cnt in enumerate(counts):
        sl = slice(start, start + cnt)
        ref = port.cascade_detect_postprocess(prop[sl], prob[sl], out[sl], cls_id=2, ratios=(cfg.ratio_h, cfg.ratio_w),
                                              org_hw=(375.0, 1242.0))
        assert dcnt[i] == len(ref), (i, dcnt[i], len(ref))
        assert np.array_equal(dets[i, : dcnt[i]], ref)
        start += cnt
