"""The several-class post-process (mscnn_detect_postprocess_classes and its Net-facade / packed / cascade forms) on the
host, without a device: the per-class loop over the restated post-process against the hand-derived vectors
(tests/golden/a15_classes_cases.json, tests/golden/make_a15_classes_vectors.py), argument checking that returns
MSCNN_ERR_INVALID before any CUDA call, and the workspace plan of N images x C classes."""
import ctypes as C
import json
import math
from pathlib import Path

import numpy as np
import pytest

from mscnn_b200 import capi

CASES = json.loads((Path(__file__).resolve().parent / "golden" / "a15_classes_cases.json").read_text())["cases"]


def _want(case):
    return [np.array(d, dtype=np.float64).reshape(-1, 5) for d in case["dets"]]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_classes_hand_vectors_oracle(case):
    import detect_classes_ref as R
    f32 = lambda k: np.array(case[k], np.float32)  # noqa: E731
    if case["kind"] == "classes":
        got = R.detect_postprocess_classes(f32("proposals_score"), f32("cls_pred"), f32("bbox_pred"), case["cls_ids"],
                                           case["det_thr"], ratios=tuple(case["ratios"]), net_hw=tuple(case["net_hw"]))
    else:
        got = R.cascade_detect_postprocess_classes(f32("proposals"), f32("cls_prob"), f32("output_bbox"),
                                                   case["cls_ids"], case["det_thr"], ratios=tuple(case["ratios"]),
                                                   org_hw=tuple(case["org_hw"]), net_hw=tuple(case["net_hw"]))
    want = _want(case)
    assert len(got) == len(want) == len(case["cls_ids"])
    for g, w in zip(got, want):
        assert g.shape == w.shape, (g, case["derivation"])
        np.testing.assert_allclose(g, w, rtol=case["tol"], atol=case["tol"], err_msg=case["derivation"])


def test_det_thr_single_precision_rounds_up():
    """The reason the fp32 comparison equals the drivers' single-vs-double one for det_thr = 0.05."""
    t = np.float32(0.05)
    assert float(t) > 0.05 and float(np.nextafter(t, np.float32(0))) < 0.05


def _cfg(num_cls=3, cap=64):
    from mscnn_b200 import net as mnet
    return mnet.kitti_detect_cfg(192, 640, max_rois=cap, num_cls=num_cls, cls_id=2)


def _classes(ids, thr=-1.0, num_ids=None):
    k = capi.DetectClasses.of(ids, thr)
    if num_ids is not None:
        k.num_ids = num_ids
    return k


BAD = {
    "no_ids": lambda: _classes([], num_ids=0),
    "too_many_ids": lambda: _classes(list(range(1, 9)), num_ids=9),
    "negative_num_ids": lambda: _classes([2], num_ids=-1),
    "id_zero": lambda: _classes([0, 2]),
    "id_above_num_cls": lambda: _classes([2, 4]),
    "duplicate_ids": lambda: _classes([2, 3, 2]),
    "nan_det_thr": lambda: _classes([2, 3], float("nan")),
    "inf_det_thr": lambda: _classes([2, 3], math.inf),
    "minus_inf_det_thr": lambda: _classes([2, 3], -math.inf),
}


@pytest.mark.parametrize("bad", sorted(BAD))
def test_invalid_class_sets_rejected_without_a_device(bad):
    """Every entry checks the class set on the host first: these return MSCNN_ERR_INVALID with any pointers, no CUDA call
    is reached (the fake pointers below would fault if one were)."""
    from mscnn_b200 import net as mnet
    L = capi.lib()
    mnet._declare(L)
    cfg, k = _cfg(), BAD[bad]()
    nb = C.c_size_t(0)
    assert L.mscnn_detect_classes_workspace_bytes(cfg, 2, k, C.byref(nb)) == capi.ERR_INVALID
    fake = [0x1000] * 5
    assert L.mscnn_detect_postprocess_classes(cfg, k, 2, *fake, 1 << 20, 0x1000, 0x1000, None, None) == capi.ERR_INVALID
    assert L.mscnn_cascade_detect_postprocess_classes(cfg, k, 2, *fake, 1 << 20, 0x1000, 0x1000, None,
                                                      None) == capi.ERR_INVALID
    assert L.mscnn_detect_postprocess_classes_packed(cfg, k, 2, *fake, 1 << 20, 0x1000, None, None) == capi.ERR_INVALID
    assert L.mscnn_net_detect_classes(None, cfg, k, 0x1000, 0x1000) == capi.ERR_INVALID
    assert L.mscnn_net_detect_cascade_classes(None, cfg, k, b"p", b"c", b"b", 0x1000, 0x1000) == capi.ERR_INVALID
    assert L.mscnn_net_detect_push_classes(None, cfg, k, 0x1000) == capi.ERR_INVALID


@pytest.mark.parametrize("n", [0, -1, 1025])
def test_batch_out_of_range_rejected_without_a_device(n):
    L = capi.lib()
    cfg, k = _cfg(), _classes([2, 3])
    nb = C.c_size_t(0)
    assert L.mscnn_detect_classes_workspace_bytes(cfg, n, k, C.byref(nb)) == capi.ERR_INVALID
    fake = [0x1000] * 5
    assert L.mscnn_detect_postprocess_classes(cfg, k, n, *fake, 1 << 20, 0x1000, 0x1000, None, None) == capi.ERR_INVALID


def test_null_class_set_and_bad_geometry_rejected_without_a_device():
    L = capi.lib()
    cfg = _cfg()
    nb = C.c_size_t(0)
    assert L.mscnn_detect_classes_workspace_bytes(cfg, 2, None, C.byref(nb)) == capi.ERR_INVALID
    fake = [0x1000] * 5
    assert L.mscnn_detect_postprocess_classes(cfg, None, 2, *fake, 1 << 20, 0x1000, 0x1000, None, None) == capi.ERR_INVALID
    geom = np.array([[1, 1, 100, 100], [1, 1, 0, 100]], np.float32)      # org_h = 0
    assert L.mscnn_detect_postprocess_classes(cfg, _classes([2, 3]), 2, *fake, 1 << 20, 0x1000, 0x1000,
                                              geom.ctypes.data, None) == capi.ERR_INVALID


def test_cfg_cls_id_is_ignored_by_the_class_entries():
    """cfg->cls_id plays no part: an out-of-range one does not make a valid class set invalid."""
    L = capi.lib()
    cfg = _cfg()
    cfg.cls_id = 0
    nb = C.c_size_t(0)
    assert L.mscnn_detect_classes_workspace_bytes(cfg, 2, _classes([2, 3]), C.byref(nb)) == capi.OK
    assert L.mscnn_detect_workspace_bytes(cfg, 2, C.byref(nb)) == capi.ERR_INVALID


@pytest.mark.parametrize("n,ids,cap", [(1, [2], 64), (3, [2, 3], 2000), (33, [3, 2], 300), (1024, [1, 2, 3], 8192),
                                       (100, [1, 2, 3, 4, 5, 6, 7, 8], 128)])
def test_workspace_is_the_single_class_plan_of_the_slots(n, ids, cap):
    L = capi.lib()
    cfg = _cfg(num_cls=8, cap=cap)
    got, ref = C.c_size_t(0), C.c_size_t(0)
    assert L.mscnn_detect_classes_workspace_bytes(cfg, n, _classes(ids), C.byref(got)) == capi.OK
    slots = n * len(ids)
    if slots <= 1024:
        assert L.mscnn_detect_workspace_bytes(cfg, slots, C.byref(ref)) == capi.OK
        assert got.value == ref.value
    else:    # beyond the single-class entry's N bound: C times the per-slot bytes of a 1024-slot plan, 256-B aligned
        assert L.mscnn_detect_workspace_bytes(cfg, 1024, C.byref(ref)) == capi.OK
        assert got.value >= ref.value * slots // 1024


def test_payload_floats_of_the_slots():
    L = capi.lib()
    assert L.mscnn_detect_payload_floats(3 * 2, 2000) == ((2 + 6 + 3) & ~3) + 6 * 2000 * 5


def test_kitti_ped_cyc_detect_cfg():
    """run_mscnn_detection.m:42-51 of the pedestrian / cyclist driver: 3 classes, ids [2 3], threshold off."""
    from mscnn_b200 import net as mnet
    cfg, k = mnet.kitti_ped_cyc_detect_cfg(768, 2560)
    assert cfg.num_cls == 3 and list(k.cls_ids[:k.num_ids]) == [2, 3] and k.det_thr <= 0
    assert list(cfg.bbox_std) == pytest.approx([0.1, 0.1, 0.2, 0.2]) and list(cfg.bbox_mean) == [0, 0, 0, 0]
    assert cfg.proposal_thr == -10.0 and cfg.nms_overlap == 0.5
    assert (cfg.ratio_h, cfg.ratio_w, cfg.org_h, cfg.org_w) == (1.0, 1.0, 768.0, 2560.0)
