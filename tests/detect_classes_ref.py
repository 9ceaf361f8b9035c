"""The per-class loop of the MATLAB drivers over the restated single-class post-process (oracle/port.py), for the tests
of the several-class post-process: examples/kitti_ped_cyc/run_mscnn_detection.m:48,93-121 runs the post-process once
per id of cls_ids, and the WIDER drivers keep only rows with prob >= det_thr before bbNms when det_thr > 0
(examples/widerface/run_mscnn_detection.m:139-143, examples/widerface/run_cascademscnn.m:130-131).

The threshold is applied to port's NMS result.  That equals filtering before NMS: greedy 'maxg' NMS only lets a kept
box suppress boxes ranked after it, and every row below the threshold ranks after every row at or above it.  The
comparison is in fp32: matcaffe returns single and the threshold is a double literal, and for the drivers' 0.05 the
two cannot differ, because single(0.05) rounds up, so no single lies in [0.05, single(0.05)).
"""
from __future__ import annotations

import numpy as np

from oracle import port


def apply_det_thr(dets: np.ndarray, det_thr: float) -> np.ndarray:
    """Rows [x y w h prob] with prob >= det_thr (fp32 compare) when det_thr > 0; all rows otherwise."""
    if det_thr <= 0:
        return dets
    return dets[dets[:, 4] >= np.float32(det_thr)]


def detect_postprocess_classes(proposals_score, cls_pred, bbox_pred, cls_ids, det_thr=-1.0, **kw) -> list[np.ndarray]:
    """One image: [K_c, 5] final detections per id of cls_ids, in that order."""
    return [apply_det_thr(port.detect_postprocess(proposals_score, cls_pred, bbox_pred, cls_id=c, **kw), det_thr)
            for c in cls_ids]


def cascade_detect_postprocess_classes(proposals, cls_prob, output_bbox, cls_ids, det_thr=-1.0,
                                       **kw) -> list[np.ndarray]:
    """One image of the cascade driver: [K_c, 5] final detections per id of cls_ids, in that order."""
    return [apply_det_thr(port.cascade_detect_postprocess(proposals, cls_prob, output_bbox, cls_id=c, **kw), det_thr)
            for c in cls_ids]
