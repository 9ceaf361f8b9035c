"""The drivers' proposal list, host side (no GPU).

(a) tests/proposals_ref.py, the numpy restatement of run_mscnn_detection.m:75-91, against hand-derived rows: a score
    exactly at proposal_thr, w or h equal to 0 and to -0.0, a NaN score, a quotient that differs from the one of the
    fp32 ratio, the dummy row of an image without proposals, and a different ratio in each axis.
(b) The specs' proposal files and the CityPersons script's default net (CITYPERSONS_BASELINE), with their source lines.
(c) drivers.write_proposals writes, byte for byte, the commented dlmwrite of the float64 rows.
(d) drivers.run refuses proposals on a cascade spec and still refuses a foreign blob triple, before any device work.
(e) mscnn_proposals_postprocess refuses a NULL pointer, N <= 0 or a bad org_hw before any CUDA call."""

import numpy as np
import pytest

import proposals_ref as R


def _row(x1, y1, x2, y2, score, img=0.0):
    return np.array([img, x1, y1, x2, y2, score], dtype=np.float32)


# ------------------------------------------------------------------------------------------------ (a) restatement
def test_threshold_is_inclusive_and_nan_is_dropped():
    rows = np.stack([_row(1, 2, 11, 22, -10.0), _row(1, 2, 11, 22, np.nextafter(np.float32(-10), np.float32(-11))),
                     _row(1, 2, 11, 22, np.nan), _row(3, 4, 5, 6, 0.5)])
    got = R.proposals(rows, -10.0, (100, 100), (100, 100))
    want = np.array([[1, 2, 10, 20, -10.0], [3, 4, 2, 2, 0.5]], dtype=np.float64)
    assert got.dtype == np.float64 and np.array_equal(got, want)


def test_zero_width_or_height_is_dropped_either_sign():
    z = np.float32(-0.0)
    rows = np.stack([_row(5, 5, 5, 9, 1.0),                       # w = 0
                     _row(5, 5, 9, 5, 1.0),                       # h = 0
                     _row(z, 5, z, 9, 1.0),                       # w = -0 - -0 = 0
                     _row(0, 5, z, 9, 1.0),                       # w = -0.0
                     _row(5, 0, 9, z, 1.0),                       # h = -0.0
                     _row(5, 5, 4, 3, 1.0)])                      # negative w and h are kept
    assert (rows[3, 3] - rows[3, 1]) == 0 and np.signbit(rows[3, 3] - rows[3, 1])
    got = R.proposals(rows, -10.0, (10, 10), (10, 10))
    assert np.array_equal(got, [[5, 5, -1, -2, 1.0]])


def test_width_is_a_single_difference():
    # x2 - x1 rounds in single (tmp(:,3) = tmp(:,3)-tmp(:,1) on matcaffe's singles): 1e8 - 0.1 is 1e8 there
    rows = np.stack([_row(0.1, 0.2, 1e8, 0.3, 1.0)])
    got = R.proposals(rows, -10.0, (1, 1), (1, 1))
    w32 = np.float32(1e8) - np.float32(0.1)
    assert got[0, 2] == float(w32) and got[0, 2] != 1e8 - float(np.float32(0.1))


def test_double_quotient_not_the_fp32_ratio_one():
    """617.3 / (2560 / 1242): the double ratio gives 299.48694720268253; the fp32 ratio widened gives another double."""
    x = np.float32(617.3)
    rows = np.stack([_row(x, 0, x + 10, 10, 0.0)])
    got = R.proposals(rows, -10.0, (768, 2560), (375, 1242))
    rd = 2560.0 / 1242.0
    assert got[0, 0] == float(x) / rd
    assert got[0, 0] != float(x) / float(np.float32(rd))
    assert got[0, 0] == 299.48694720268253


def test_dummy_row_of_an_empty_image_is_dropped():
    dummy = np.zeros((1, 6), np.float32)          # box_output_layer.cpp: a zero proposals_score row
    got = R.proposals(dummy, -10.0, (768, 2560), (375, 1242))
    assert got.shape == (0, 5) and got.dtype == np.float64


def test_each_axis_has_its_own_ratio():
    rows = np.stack([_row(100, 100, 300, 500, 2.0)])
    got = R.proposals(rows, -5.0, (768, 2560), (384, 640))           # ratios (2, 4)
    assert np.array_equal(got, [[25.0, 50.0, 50.0, 200.0, 2.0]])
    assert R.ratios((768, 2560), (384, 640)) == (2.0, 4.0)


def test_split_rows_by_counts():
    rows = np.arange(5 * 6, dtype=np.float32).reshape(5, 6)
    parts = R.split_rows(rows, [2, 0, 3])
    assert [len(p) for p in parts] == [2, 0, 3] and np.array_equal(parts[2], rows[2:])


# ----------------------------------------------------------------------------------------------------- (b) specs
def test_proposal_files_and_the_baseline_spec():
    from mscnn_b200 import drivers as D
    for s in (D.KITTI_CAR, D.KITTI_PED_CYC, D.CALTECH):
        assert s.proposals_file == "{comp_id}.txt" and not s.cascade
        assert "proposals_file" in s.source and "proposals" in s.source
    assert D.KITTI_CAR.source["proposals_file"].startswith(":162")
    assert D.KITTI_PED_CYC.source["proposals_file"].startswith(":162")
    assert D.CALTECH.source["proposals_file"].startswith(":169")
    for s in (D.KITTI_CAR_CASCADE, D.CITYPERSONS, D.CITYPERSONS_BASELINE):
        assert s.proposals_file is None
    b = D.CITYPERSONS_BASELINE
    assert D.SPECS["citypersons_baseline"] is b
    assert b.script == "examples/citypersons/run_cascademscnn.m"
    assert b.net_hw == (1344, 2688) and b.num_cls == 2 and b.cls_ids == (2,) and b.cascade and b.obj_names is None
    assert b.blobs == ("proposals", "cls_prob_1st", "output_bbox_1st")
    assert b.det_thr == -1.0 and b.nms_overlap == 0.5 and b.proposal_thr is None and b.bbox_stds is None
    assert b.result_files == ("{comp_id}_1st_results.txt",) and b.index_across_groups
    fields = {"script", "net_hw", "num_cls", "cls_ids", "obj_names", "cascade", "blobs", "bbox_stds", "proposal_thr",
              "nms_overlap", "det_thr", "result_files", "index_across_groups", "proposals_file"}
    assert fields <= set(b.source), fields - set(b.source)
    assert b.source["blobs"].startswith(":36-41") and b.source["script"].startswith(":11")
    assert [p.name for p in b.result_paths("detections", "mscnn_8s_1344_2x_pretrained")] == \
        ["mscnn_8s_1344_2x_pretrained_1st_results.txt"]


# ------------------------------------------------------------------------------------------------- (c) the file
def test_write_proposals_is_the_commented_dlmwrite(tmp_path):
    from mscnn_b200 import drivers as D
    props = [np.array([[1.00005, 2.5, 123.455, 40.0, -3.25],
                       [0.0, -0.5, 1e-7, 123456.0, 0.9999949]], dtype=np.float64),
             np.zeros((0, 5), np.float64),
             np.array([[10.0, 20.0, 30.0, 40.0, 1.0]])]
    # %.5g of the double and of its float32 rounding differ for 1.00005 ("1.0001" / "1") and 123.455
    assert "%.5g" % 1.00005 != "%.5g" % float(np.float32(1.00005))
    assert "%.5g" % 123.455 != "%.5g" % float(np.float32(123.455))
    want = ("1,1.0001,2.5,123.45,40,-3.25\n"
            "1,0,-0.5,1e-07,1.2346e+05,0.99999\n"
            "3,10,20,30,40,1\n").encode()
    p = D.write_proposals(tmp_path / "proposals", D.KITTI_CAR, "mscnn_8s_768", props)
    assert p == tmp_path / "proposals" / "mscnn_8s_768.txt"
    assert p.read_bytes() == want
    assert p.read_bytes() == R.dlmwrite(props)
    p = D.write_proposals(tmp_path / "part", D.CALTECH, "c", props[2:], first_index=3)
    assert p.read_bytes() == b"3,10,20,30,40,1\n"
    assert D.write_proposals(tmp_path / "none", D.KITTI_PED_CYC, "c", [np.zeros((0, 5))]).read_bytes() == b""
    for s in (D.KITTI_CAR_CASCADE, D.CITYPERSONS, D.CITYPERSONS_BASELINE):
        with pytest.raises(ValueError):
            D.write_proposals(tmp_path, s, "c", props)


# ------------------------------------------------------------------------------------------------ (d) refusals
def test_run_refuses_proposals_on_cascade_specs_and_foreign_blobs():
    import dataclasses
    from mscnn_b200 import drivers as D
    frames = [np.zeros((8, 8, 3), np.uint8)]
    for s in (D.KITTI_CAR_CASCADE, D.CITYPERSONS, D.CITYPERSONS_BASELINE):
        with pytest.raises(ValueError, match="no proposal list"):
            D.run(object(), frames, s, proposals=True)
    for blobs in (("proposals_2nd", "cls_prob_2nd", "output_bbox_2nd"), ("proposals", "cls_prob_1st", "output_bbox_3rd"),
                  ("proposals_3rd", "cls_prob_3rd", "output_bbox_1st")):
        foreign = dataclasses.replace(D.CITYPERSONS, blobs=blobs)
        for prop in (False, True):
            with pytest.raises(ValueError, match="unsupported cascade blobs"):
                D.run(object(), frames, foreign, proposals=prop)
    from mscnn_b200 import widerface
    with pytest.raises(ValueError):
        widerface.run(object(), frames, ["a"], cascade=True, proposals=True)


# ------------------------------------------------------------------------------------------------ (e) the C entry
def test_c_entry_refuses_bad_arguments_without_cuda():
    from mscnn_b200 import capi, net as mnet
    L = capi.lib()
    INV = capi.ERR_INVALID
    cfg = mnet.kitti_detect_cfg(192, 640)
    fake = 0x1000                                       # never dereferenced on these paths
    hw = np.array([[375, 1242], [370, 1224]], np.int32)
    f = L.mscnn_proposals_postprocess
    assert f(None, 2, fake, fake, 192, 640, hw.ctypes.data, fake, fake, None) == INV
    for n in (0, -1):
        assert f(cfg, n, fake, fake, 192, 640, hw.ctypes.data, fake, fake, None) == INV
    for k in range(4):                                  # each device pointer NULL in turn
        p = [fake] * 4
        p[k] = None
        assert f(cfg, 2, p[0], p[1], 192, 640, hw.ctypes.data, p[2], p[3], None) == INV, k
    for nh, nw in ((0, 640), (192, 0), (-1, 640)):
        assert f(cfg, 2, fake, fake, nh, nw, hw.ctypes.data, fake, fake, None) == INV
    for bad in ([[375, 1242], [0, 1224]], [[375, -5], [370, 1224]]):
        b = np.array(bad, np.int32)
        assert f(cfg, 2, fake, fake, 192, 640, b.ctypes.data, fake, fake, None) == INV, bad
    cfg0 = mnet.kitti_detect_cfg(192, 640)
    cfg0.org_h = 0.0                                    # org_hw NULL: the cfg's sizes must be positive
    assert f(cfg0, 2, fake, fake, 192, 640, None, fake, fake, None) == INV
    cfg0 = mnet.kitti_detect_cfg(192, 640)
    cfg0.max_rois_per_image = 0
    assert f(cfg0, 2, fake, fake, 192, 640, hw.ctypes.data, fake, fake, None) == INV
    mnet._declare(L)
    assert L.mscnn_net_proposals(None, cfg, fake, fake) == INV
