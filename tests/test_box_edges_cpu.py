"""The edge cases of tests/box_edge_cases.py hit the edge each one claims, measured with the oracle alone (no GPU): a
builder change that loses its edge fails here instead of passing quietly on the device."""
from __future__ import annotations

import numpy as np
import pytest

import box_edge_cases as E
from oracle import port

F32 = np.float32
BOX = E.box_cases()
DET = E.det_cases()


def _rows_xywh(rois_score):
    """[img x1 y1 x2 y2 score] rows -> [img x y w h score] (exact for the integer boxes of the builders)."""
    r = rois_score.astype(np.float64).copy()
    r[:, 3] -= r[:, 1]
    r[:, 4] -= r[:, 2]
    return r


def _key(img, box):
    return (int(img), *[float(v) for v in box[:4]])


def _sorted_and_kept(case, n):
    """Rows of image n in the oracle's ranking (NMS off: no IoU exceeds 1) and the keys of the rows it keeps."""
    k = case.cfg["max_nms_num"]
    _, srt, _, _ = case.oracle(iou_thr=1.0, max_post_nms_num=0)
    _, kept, _, _ = case.oracle(max_post_nms_num=0)
    srt = _rows_xywh(srt)
    srt = srt[srt[:, 0] == n]
    kept = _rows_xywh(kept)
    keys = {_key(r[0], r[1:5]) for r in kept}
    assert len(srt) <= k
    return srt, keys


@pytest.mark.parametrize("case", BOX, ids=[c.name for c in BOX])
def test_box_case_hits_its_edge(case):
    print(f"{case.name}: {case.edge}")
    c = case.claims
    rois, sc, per, true = case.oracle()
    assert int(per.sum()) == true
    xywh = _rows_xywh(sc) if true else sc[:0].astype(np.float64)
    kept = {_key(r[0], r[1:5]) for r in xywh}
    if "valid" in c:
        # NMS off: the sorted list holds min(valid, K) boxes, and min(valid, K + 1) when K is one larger
        k = case.cfg["max_nms_num"]
        for kk in (k, k + 1):
            _, _, p, _ = case.oracle(iou_thr=1.0, max_post_nms_num=0, max_nms_num=kk)
            assert list(p) == [min(v, kk) for v in c["valid"]], (kk, list(p), c["valid"])
    if c.get("suppresses"):
        _, _, p, _ = case.oracle(iou_thr=1.0, max_post_nms_num=0)
        assert true < int(p.sum()), "NMS suppresses nothing"
    if "tie_pairs" in c:
        thr = F32(case.cfg["iou_thr"])
        for n, a, b in c["tie_pairs"]:
            iou = F32(port.box_iou(a, b, case.cfg["nms_type"]))
            assert iou == F32(c["tie_value"])
            assert (iou > thr) != c["tie_kept"], (iou, thr)
            assert _key(n, a) in kept
            assert (_key(n, b) in kept) == c["tie_kept"], (a, b)
    if c.get("chain_edges"):
        srt, keys = _sorted_and_kept(case, 0)
        flags = [_key(0, r[1:5]) in keys for r in srt]
        assert len(set(_key(0, r[1:5]) for r in srt)) == len(srt)
        starts_suppressed = passes = 0
        for b in range(1, (len(srt) + 63) // 64):
            prev, first = srt[64 * b - 1], srt[64 * b]
            overlap = port.box_iou(prev[1:5], first[1:5]) > F32(case.cfg["iou_thr"])
            starts_suppressed += flags[64 * b - 1] and not flags[64 * b] and overlap
            passes += (not flags[64 * b - 1]) and flags[64 * b] and overlap
        assert starts_suppressed >= 2 and passes >= 2, (starts_suppressed, passes)
    if "k_tie" in c:
        k = c["k_tie"]
        _, s, _, _ = case.oracle(iou_thr=1.0, max_nms_num=k + 1)
        assert len(s) == k + 1 and s[k - 1, 5] == s[k, 5], "the K-th and (K+1)-th scores differ"
        if k > 1:
            assert s[k - 2, 5] == s[k - 1, 5] or k - 1 == 0
        if c["signed_zero"]:
            _, s, _, _ = case.oracle(iou_thr=1.0, max_nms_num=len(s) + 200)
            bits = s[:, 5].view(np.uint32)
            neg, pos = np.flatnonzero(bits == 0x80000000), np.flatnonzero(bits == 0)
            assert len(neg) and len(pos) and neg.min() < pos.max() and neg.min() < k <= pos.max()
            # the oracle's top K takes -0 boxes that a +0-first ranking would leave out
            assert (bits[:k] == 0x80000000).any() and (bits[k:] == 0).any()
    if "kept_uncapped" in c:
        _, _, p, _ = case.oracle(max_post_nms_num=0)
        mp = case.cfg["max_post_nms_num"]
        assert list(p) == c["kept_uncapped"]
        assert list(per) == [min(v, mp) for v in c["kept_uncapped"]]
    if true == 0:
        assert rois.tolist() == [[0.0, 1.0, 1.0, 10.0, 10.0]] and not sc.any()


def test_box_cases_cover_the_counts():
    names = {c.name for c in BOX}
    for k in E.COUNT_KS:
        for v in {0, k - 1, k, k + 1, 2 * k + 37}:
            assert f"count_K{k}_valid{v}" in names
    modes = {c.cfg["nms_type"] for c in BOX if "tie_pairs" in c.claims}
    assert modes == {"IOU", "IOMU", "IOFU"}
    assert {c.cfg["max_post_nms_num"] for c in BOX} >= {63, 64, 65, 128}
    runs = {(c.claims["k_tie"], c.claims["signed_zero"]) for c in BOX if "k_tie" in c.claims}
    assert len(runs) >= 6 and any(s for _, s in runs)
    empties = [c.claims["valid"] for c in BOX if c.name.startswith("batch_")]
    assert [0] in empties and any(v[0] == 0 for v in empties if len(v) == 3)
    assert any(v[1] == 0 < v[0] for v in empties if len(v) == 3) and any(v[2] == 0 < v[0] for v in empties if len(v) == 3)


def test_exp_arguments_are_unambiguous():
    assert E.exp_unambiguous(0.0)
    for v in E.LOGITS:
        assert E.exp_unambiguous(v), v
    assert E.exp_unambiguous(E.logf(2.0)) and E.exp_unambiguous(E.logf(0.5))


def _sorted_probs(case, n, cls_id):
    return case.oracle(n, cls_id, overlap=1.0, det_thr=-1.0)


@pytest.mark.parametrize("case", DET, ids=[c.name for c in DET])
def test_det_case_hits_its_edge(case):
    print(f"{case.name}: {case.edge}")
    c = case.claims
    refs = [[case.oracle(n, cid) for cid in case.cls_ids] for n in range(case.n)]
    for n in range(case.n):
        for d in refs[n]:
            assert len(d) <= case.max_rois
    assert any(len(d) for r in refs for d in r)
    if "tie_pairs" in c:
        ov = F32(case.overlap)
        for n, a, b in c["tie_pairs"]:
            o = E.bbnms_overlap(a, b)
            assert o == c["tie_value"] and (o > float(ov)) != c["tie_kept"]
            got = {tuple(float(v) for v in r[:4]) for r in refs[n][0]}
            assert tuple(map(float, a)) in got and (tuple(map(float, b)) in got) == c["tie_kept"]
    if c.get("prob_tie_edges"):
        hits = 0
        for n in range(case.n):
            s = _sorted_probs(case, n, case.cls_ids[0])
            hits += sum(s[64 * b - 1, 4] == s[64 * b, 4] for b in range(1, (len(s) + 63) // 64))
        assert hits >= 2
    if c.get("signed_zero"):
        s = _sorted_probs(case, 0, case.cls_ids[0])
        bits = s[:, 4].view(np.uint32)
        neg, pos = np.flatnonzero(bits == 0x80000000), np.flatnonzero(bits == 0)
        assert len(neg) and len(pos) and neg.min() < pos.max() and pos.min() < neg.max(), "+0 and -0 not interleaved"
    if "rows" in c:
        assert list(case.counts) == c["rows"]
        assert max(c["rows"]) == case.max_rois
    if c.get("prob_ties"):
        s = _sorted_probs(case, int(np.argmax(case.counts)), case.cls_ids[0])
        assert (s[1:, 4] == s[:-1, 4]).any()
        if len(s) > 64:
            assert any(s[64 * b - 1, 4] == s[64 * b, 4] for b in range(1, (len(s) + 63) // 64))
    if c.get("det_thr_hit"):
        assert case.det_thr > 0
        hit = [(d[:, 4] == F32(case.det_thr)).any() for r in refs for d in r]
        assert any(hit)
        full = [case.oracle(n, cid, det_thr=-1.0) for n in range(case.n) for cid in case.cls_ids]
        assert sum(map(len, full)) > sum(len(d) for r in refs for d in r), "det_thr drops nothing"


def test_det_cases_cover_the_counts():
    caps = {c.max_rois for c in DET}
    assert caps >= {64, 65, 2048, 8192}
    assert any(c.cascade for c in DET) and any(not c.cascade for c in DET)
    for c in DET:
        if "rows" in c.claims:
            assert c.max_rois in c.counts
