"""Hand-derived known answers for the post-process of SEVERAL classes with the drivers' detection threshold (the
per-class loop of examples/kitti_ped_cyc/run_mscnn_detection.m:48,93-121 and the `det_thr` filter of
examples/widerface/run_mscnn_detection.m:57,139-143 / examples/widerface/run_cascademscnn.m:67,130-131).  This file
writes tests/golden/a15_classes_cases.json; every case carries its derivation.  Like make_a15_vectors.py it imports
nothing from the repo: the expected numbers are literals.

    python tests/golden/make_a15_classes_vectors.py

Conventions shared by every case: bbox deltas are zero, so a decoded box is its proposal in [x y w h]
(run_mscnn_detection.m:104-109: ctr = x + 0.5 w, tx = 0 * w + ctr - w / 2 = x, tw = w * exp(0) = w); the image is
large enough that the clip of :114-115 is inactive; NMS is bbNms 'maxg' with overlap 0.5 ('union' denominator).
`dets[c]` lists the final rows [x y w h prob] of class cls_ids[c], in the order the caller gave the ids.
"""
import json
import math
from pathlib import Path

cases = []
ln3 = math.log(3.0)

# three classes (bg, ped, cyc) like the KITTI pedestrian / cyclist nets
A = [0, 0, 0, 100, 100]        # [img x1 y1 x2 y2]
B = [0, 20, 0, 120, 100]       # overlaps A: iw = 80, o = 8000 / (20000 - 8000) = 0.667
Cc = [0, 200, 200, 300, 300]   # disjoint from both
props = [A + [1.0], B + [1.0], Cc + [1.0]]
logits = [[0.0, ln3, 0.0], [0.0, 0.0, ln3], [0.0, 0.0, 0.0]]
zero_deltas = [[0.0] * 12] * 3
p_hi, p_lo, p_third = 3.0 / 5.0, 1.0 / 5.0, 1.0 / 3.0
per_class_derivation = (
    "Softmax per row (run_mscnn_detection.m:101-103): A logits [0 ln3 0] -> exp [1 3 1] -> p = [1/5 3/5 1/5]; "
    "B [0 0 ln3] -> [1/5 1/5 3/5]; C [0 0 0] -> [1/3 1/3 1/3].  A and B overlap 8000 / 12000 = 0.667 > 0.5; C is "
    "disjoint.  Class 2 (ped): ranked A 3/5, C 1/3, B 1/5 -> A suppresses B -> [A, C].  Class 3 (cyc): ranked B 3/5, "
    "C 1/3, A 1/5 -> B suppresses A -> [B, C].  The same ROI set keeps different rows per class, which is why the "
    "driver runs bbNms once per id (:93-121).")
cases.append(dict(
    name="per_class_nms_keeps_different_rows",
    kind="classes", num_cls=3, cls_ids=[2, 3], det_thr=-1, net_hw=[400, 400], ratios=[1.0, 1.0],
    proposals_score=props, cls_pred=logits, bbox_pred=zero_deltas,
    dets=[[[0.0, 0.0, 100.0, 100.0, p_hi], [200.0, 200.0, 100.0, 100.0, p_third]],
          [[20.0, 0.0, 100.0, 100.0, p_hi], [200.0, 200.0, 100.0, 100.0, p_third]]],
    tol=2e-6, derivation=per_class_derivation))
cases.append(dict(
    name="class_order_is_the_callers",
    kind="classes", num_cls=3, cls_ids=[3, 2], det_thr=-1, net_hw=[400, 400], ratios=[1.0, 1.0],
    proposals_score=props, cls_pred=logits, bbox_pred=zero_deltas,
    dets=[[[20.0, 0.0, 100.0, 100.0, p_hi], [200.0, 200.0, 100.0, 100.0, p_third]],
          [[0.0, 0.0, 100.0, 100.0, p_hi], [200.0, 200.0, 100.0, 100.0, p_third]]],
    tol=2e-6, derivation="The rows of case per_class_nms_keeps_different_rows with cls_ids = [3 2]: output slot 0 is "
                         "class 3 ([B, C]), slot 1 class 2 ([A, C]); the ids are taken in the caller's order."))
cases.append(dict(
    name="nan_logit_row_dropped_in_every_class",
    kind="classes", num_cls=3, cls_ids=[2, 3], det_thr=-1, net_hw=[400, 400], ratios=[1.0, 1.0],
    proposals_score=props + [[0, 200, 200, 300, 300, 5.0]],
    cls_pred=logits + [[0.0, float("nan"), 0.0]], bbox_pred=zero_deltas + [[0.0] * 12],
    dets=[[[0.0, 0.0, 100.0, 100.0, p_hi], [200.0, 200.0, 100.0, 100.0, p_third]],
          [[20.0, 0.0, 100.0, 100.0, p_hi], [200.0, 200.0, 100.0, 100.0, p_third]]],
    tol=2e-6, derivation="A fourth row, the box of C, whose class-2 logit is NaN: sum(exp) = NaN, so prob = NaN for "
                         "EVERY class (:101-103), and bbNms drops it (bbNms.m:82 kp = bbs(:,5) > -inf is false for "
                         "NaN) before it can suppress C.  Both classes equal case per_class_nms_keeps_different_rows."))

# two classes, detection threshold
R1 = [0, 0, 0, 50, 50]          # logits [0 0]   -> p = [1/2 1/2] exactly
R2 = [0, 100, 0, 150, 50]       # logits [0 ln3] -> p = [1/4 3/4]
R3 = [0, 200, 0, 250, 50]       # logits [ln3 0] -> p = [3/4 1/4]
thr_props = [R1 + [0.0], R2 + [0.0], R3 + [0.0]]
thr_logits = [[0.0, 0.0], [0.0, ln3], [ln3, 0.0]]
thr_deltas = [[0.0] * 8] * 3
thr_derivation = (
    "Three disjoint boxes (no suppression), two classes.  exp(0) = 1 and 1 / (1 + 1) = 0.5 are exact in single, so R1 "
    "has prob 0.5 in both classes, EQUAL to det_thr = 0.5 (also exact): the driver keeps prob >= det_thr "
    "(widerface/run_mscnn_detection.m:139-141), so R1 stays.  R2: p = [1/4 3/4]; R3: p = [3/4 1/4].  Class 2: R2 "
    "0.75 and R1 0.5 stay, R3 0.25 < 0.5 goes.  Class 1: R3 0.75, R1 0.5; R2 goes.  Rows by descending prob.")
cases.append(dict(
    name="prob_equal_to_det_thr_is_kept",
    kind="classes", num_cls=2, cls_ids=[2, 1], det_thr=0.5, net_hw=[400, 400], ratios=[1.0, 1.0],
    proposals_score=thr_props, cls_pred=thr_logits, bbox_pred=thr_deltas,
    dets=[[[100.0, 0.0, 50.0, 50.0, 0.75], [0.0, 0.0, 50.0, 50.0, 0.5]],
          [[200.0, 0.0, 50.0, 50.0, 0.75], [0.0, 0.0, 50.0, 50.0, 0.5]]],
    tol=2e-6, derivation=thr_derivation))
for thr in (0.0, -1.0):
    cases.append(dict(
        name=f"det_thr_{'zero' if thr == 0 else 'minus_one'}_is_off",
        kind="classes", num_cls=2, cls_ids=[2, 1], det_thr=thr, net_hw=[400, 400], ratios=[1.0, 1.0],
        proposals_score=thr_props, cls_pred=thr_logits, bbox_pred=thr_deltas,
        dets=[[[100.0, 0.0, 50.0, 50.0, 0.75], [0.0, 0.0, 50.0, 50.0, 0.5], [200.0, 0.0, 50.0, 50.0, 0.25]],
              [[200.0, 0.0, 50.0, 50.0, 0.75], [0.0, 0.0, 50.0, 50.0, 0.5], [100.0, 0.0, 50.0, 50.0, 0.25]]],
        tol=2e-6, derivation=f"The rows of case prob_equal_to_det_thr_is_kept with det_thr = {thr}: the drivers "
                             "filter only `if (det_thr > 0)` (widerface/run_mscnn_detection.m:139), so nothing is "
                             "dropped and every class keeps all three disjoint rows, by descending prob."))

# cascade driver (run_cascademscnn.m:96-131): boxes come from output_bbox with the "+ 1" extent convention
cases.append(dict(
    name="cascade_classes_with_det_thr",
    kind="cascade_classes", num_cls=3, cls_ids=[2, 3], det_thr=0.05, net_hw=[400, 400], ratios=[1.0, 1.0],
    org_hw=[400, 400],
    proposals=[[0, 0, 0, 9, 9], [0, 100, 100, 109, 109], [0, 50, 50, 59, 59]],
    cls_prob=[[0.5, 0.45, 0.05], [0.9, 0.06, 0.04], [0.2, 0.3, 0.5]],
    output_bbox=[[0, 0, 0, 9, 9], [0, 100, 100, 109, 109], [0, 50, 50, 59, 59]],
    dets=[[[0.0, 0.0, 10.0, 10.0, 0.45], [50.0, 50.0, 10.0, 10.0, 0.3], [100.0, 100.0, 10.0, 10.0, 0.06]],
          [[50.0, 50.0, 10.0, 10.0, 0.5], [0.0, 0.0, 10.0, 10.0, 0.05]]],
    tol=2e-6,
    derivation="Unit ratios, so [x1 y1 x2 y2] stay and w = x2 - x1 + 1 = 10 (run_cascademscnn.m:101-106); the three "
               "boxes are disjoint.  det_thr = 0.05 > 0: keep prob >= det_thr (widerface/run_cascademscnn.m:130-131).  "
               "matcaffe returns single and the threshold is a double literal; single(0.05) rounds UP, so no single "
               "lies in [0.05, single(0.05)) and comparing in single gives the same answer: the class-3 probability "
               "0.05 of row 1 (stored as single(0.05)) equals the threshold and stays.  Class 2: 0.45, 0.3, 0.06 all "
               "stay.  Class 3: row 3 0.5 and row 1 0.05 stay, row 2 0.04 goes."))

out = Path(__file__).resolve().parent / "a15_classes_cases.json"
out.write_text(json.dumps(dict(source="hand-derived from kitti_ped_cyc/run_mscnn_detection.m:48,93-121 and the "
                                      "det_thr filter of the WIDER drivers; see make_a15_classes_vectors.py",
                               cases=cases), indent=1))
print(f"{len(cases)} cases -> {out}")
