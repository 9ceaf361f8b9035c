"""BoxOutput and the final-detection post-process on the device against oracle.port, bit for bit, on the edge cases of
tests/box_edge_cases.py: IoU and bbNms overlaps exactly on the threshold, greedy chains across the 64-box blocks of the
NMS kernels, equal scores across the top-K cut (+-0 and +inf included), max_nms_num up to the 8192 cap against valid
counts around it, max_post_nms_num at the block sizes, empty images, NaN / inf map values, per-image row counts up to
max_rois_per_image 8192.  The geometry of every case is exact, so nothing is compared with a tolerance.

Zero scores compare by value: the device ranks -0 and +0 as equal (as the reference's std::greater and MATLAB's sort do)
and writes every zero score as +0."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

import box_edge_cases as E

pytestmark = pytest.mark.gpu

BOX = E.box_cases()
DET = E.det_cases()


def _same_rows(got, ref, score_col=None):
    """Bit-exact rows; a zero score only has to be zero."""
    got, ref = np.array(got, np.float32), np.array(ref, np.float32)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if score_col is not None:
        gz, rz = got[:, score_col] == 0, ref[:, score_col] == 0
        assert np.array_equal(gz, rz), np.flatnonzero(gz != rz)[:10]
        got[gz, score_col] = 0.0
        ref[rz, score_col] = 0.0
    bad = np.flatnonzero((got.view(np.uint32) != ref.view(np.uint32)).any(axis=1))
    assert not len(bad), f"{len(bad)} rows differ, first {bad[0]}: device {got[bad[0]]} vs oracle {ref[bad[0]]}"


def _box_cfg(case, **over):
    from mscnn_b200 import ops
    a = case.oracle_args(**over)
    shapes = [(m.shape[1], m.shape[2], m.shape[3]) for m in case.maps]
    return ops.make_box_cfg(shapes, a["field_w"], a["field_h"], a["downsample_rate"], a["fg_thr"], a["iou_thr"],
                            a["nms_type"], a["field_whr"], a["field_xyr"], a["min_size"], a["max_nms_num"],
                            a["max_post_nms_num"])


def _box_device(cuda, case, maps=None):
    from mscnn_b200 import ops
    rois, rois_score, num_out = ops.box_output_forward(_box_cfg(case), [torch.from_numpy(m).to(cuda)
                                                                        for m in (maps or case.maps)])
    torch.cuda.synchronize()
    no = num_out.cpu().numpy()
    return rois[:no[0]].cpu().numpy(), rois_score[:no[0]].cpu().numpy(), no


def _compare_box(got, ref):
    g_rois, g_sc, g_no = got
    rois, sc, per, true = ref
    assert g_no[1] == true and g_no[0] == max(true, 1), (g_no[:2], true)
    assert list(g_no[2:]) == list(per), (list(g_no[2:]), list(per))
    _same_rows(g_rois, rois)
    _same_rows(g_sc, sc, score_col=5)


@pytest.mark.parametrize("case", BOX, ids=[c.name for c in BOX])
def test_box_output_edge_case(cuda, case):
    _compare_box(_box_device(cuda, case), case.oracle())


def _det_cfg(case, cls_id=None):
    from mscnn_b200 import capi
    cfg = capi.DetectCfg()
    cfg.num_cls, cfg.cls_id = case.num_cls, cls_id or case.cls_ids[0]
    for k, v in enumerate([0.1, 0.1, 0.2, 0.2]):
        cfg.bbox_std[k], cfg.bbox_mean[k] = v, 0.0
    cfg.proposal_thr, cfg.nms_overlap = -10.0, case.overlap
    cfg.ratio_h = cfg.ratio_w = 1.0
    cfg.org_h, cfg.org_w = case.org_hw
    cfg.max_rois_per_image = case.max_rois
    return cfg


def _det_inputs(cuda, case):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(cuda) for a in (case.prop, case.cls, case.bbox, case.num_out())]


@pytest.mark.parametrize("case", DET, ids=[c.name for c in DET])
def test_detect_single_class_edge_case(cuda, case):
    from mscnn_b200 import ops
    dev = _det_inputs(cuda, case)
    f = ops.cascade_detect_postprocess if case.cascade else ops.detect_postprocess
    for cid in case.cls_ids:
        dets, cnt = f(_det_cfg(case, cid), case.n, *dev)
        torch.cuda.synchronize()
        dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
        for n in range(case.n):
            ref = case.oracle(n, cid, det_thr=-1.0)
            assert cnt[n] == len(ref), (n, cid, int(cnt[n]), len(ref))
            _same_rows(dets[n, :cnt[n]], ref, score_col=4)


@pytest.mark.parametrize("case", DET, ids=[c.name for c in DET])
def test_detect_classes_edge_case(cuda, case):
    """Every class slot of the several-class entry, with the case's detection threshold; and the packed payload."""
    from mscnn_b200 import capi, ops, parallel
    dev = _det_inputs(cuda, case)
    cfg = _det_cfg(case)
    k = capi.DetectClasses.of(case.cls_ids, case.det_thr)
    f = ops.cascade_detect_postprocess_classes if case.cascade else ops.detect_postprocess_classes
    dets, cnt = f(cfg, k, case.n, *dev)
    packed = None if case.cascade else ops.detect_postprocess_classes_packed(cfg, k, case.n, *dev)
    torch.cuda.synchronize()
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    slots = None if packed is None else parallel.unpack_payload(packed, 1, case.n * len(case.cls_ids), case.max_rois)
    for n in range(case.n):
        for c, cid in enumerate(case.cls_ids):
            ref = case.oracle(n, cid)
            assert cnt[n, c] == len(ref), (n, cid, int(cnt[n, c]), len(ref))
            _same_rows(dets[n, c, :cnt[n, c]], ref, score_col=4)
            if slots is not None:
                _same_rows(slots[n * len(case.cls_ids) + c], ref, score_col=4)


def _case(name, cases):
    return next(c for c in cases if c.name == name)


def test_box_output_workspace_and_untouched_rows(cuda):
    """Through the C entry: a workspace of 0xFF bytes and NaN outputs; rows past num_out[0] stay NaN; a second,
    different input through the same workspace equals the oracle and a run on a fresh workspace."""
    from mscnn_b200 import capi
    first, second = _case("count_K2049_valid4135", BOX), _case("count_K2048_valid4133", BOX)
    assert [m.shape for m in first.maps] == [m.shape for m in second.maps]
    cfg = _box_cfg(first)
    n = first.n
    nbytes = C.c_size_t(0)
    capi.check(capi.lib().mscnn_box_output_workspace_bytes(cfg, n, C.byref(nbytes)))
    ws = torch.full((nbytes.value,), 0xFF, dtype=torch.uint8, device=cuda)
    cap = n * cfg.max_nms_num
    for case in (first, second):
        maps = [torch.from_numpy(m).to(cuda) for m in case.maps]
        rois = torch.full((cap, 5), float("nan"), device=cuda)
        rois_score = torch.full((cap, 6), float("nan"), device=cuda)
        num_out = torch.full((2 + n,), -1, dtype=torch.int32, device=cuda)
        ptrs = (C.c_void_p * len(maps))(*[m.data_ptr() for m in maps])
        capi.check(capi.lib().mscnn_box_output_forward(cfg, n, ptrs, capi.ptr(ws), nbytes.value, capi.ptr(rois),
                                                       capi.ptr(rois_score), capi.ptr(num_out), None))
        torch.cuda.synchronize()
        no = num_out.cpu().numpy()
        rows = int(no[0])
        r, s = rois.cpu().numpy(), rois_score.cpu().numpy()
        assert np.isnan(r[rows:]).all() and np.isnan(s[rows:]).all()
        got = (r[:rows], s[:rows], no)
        _compare_box(got, port_box(case, first))
        fresh = _box_device(cuda, first, maps=case.maps)
        assert np.array_equal(fresh[2], no)
        assert np.array_equal(fresh[0].view(np.uint32), got[0].view(np.uint32))
        assert np.array_equal(fresh[1].view(np.uint32), got[1].view(np.uint32))


def port_box(case, cfg_case):
    """The oracle on `case`'s maps with `cfg_case`'s configuration."""
    from oracle import port
    return port.box_output(case.maps, **cfg_case.oracle_args())


def test_detect_workspace_and_untouched_rows(cuda):
    """The same for mscnn_detect_postprocess and mscnn_cascade_detect_postprocess: rows past det_counts stay NaN."""
    from mscnn_b200 import capi
    for first, second in (("mscnn_rows_2048", "mscnn_rows_65"), ("cascade_count_2048", "cascade_count_8192")):
        a, b = _case(first, DET), _case(second, DET)
        cfg = _det_cfg(b if b.max_rois > a.max_rois else a)
        n = max(a.n, b.n)
        nbytes = C.c_size_t(0)
        capi.check(capi.lib().mscnn_detect_workspace_bytes(cfg, n, C.byref(nbytes)))
        ws = torch.full((nbytes.value,), 0xFF, dtype=torch.uint8, device=cuda)
        entry = capi.lib().mscnn_cascade_detect_postprocess if a.cascade else capi.lib().mscnn_detect_postprocess
        for case in (a, b):
            dev = _det_inputs(cuda, case)
            dets = torch.full((case.n, cfg.max_rois_per_image, 5), float("nan"), device=cuda)
            cnt = torch.full((case.n,), -1, dtype=torch.int32, device=cuda)
            capi.check(entry(cfg, case.n, *map(capi.ptr, dev), capi.ptr(ws), nbytes.value, capi.ptr(dets),
                             capi.ptr(cnt), None))
            torch.cuda.synchronize()
            d, k = dets.cpu().numpy(), cnt.cpu().numpy()
            for i in range(case.n):
                ref = case.oracle(i, cfg.cls_id, det_thr=-1.0)
                assert k[i] == len(ref)
                _same_rows(d[i, :k[i]], ref, score_col=4)
                assert np.isnan(d[i, k[i]:]).all()


def test_repeat_launches_give_the_same_bits(cuda):
    from mscnn_b200 import ops
    case = _case("count_K8192_valid16421", BOX)
    a, b = _box_device(cuda, case), _box_device(cuda, case)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))
    case = _case("cascade_count_8192", DET)
    dev = _det_inputs(cuda, case)
    cfg = _det_cfg(case)
    d1, c1 = ops.cascade_detect_postprocess(cfg, case.n, *dev)
    d2, c2 = ops.cascade_detect_postprocess(cfg, case.n, *dev)
    torch.cuda.synchronize()
    assert torch.equal(c1, c2) and torch.equal(d1.view(torch.int32), d2.view(torch.int32))
