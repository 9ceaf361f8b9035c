"""The drivers' proposal list, restated in numpy from the MATLAB lines it comes from
(examples/kitti_car/run_mscnn_detection.m:75-91; the same lines in kitti_ped_cyc, caltech :80-96 and
widerface :93-109):

    tmp = squeeze(outputs{3}); tmp = tmp'; tmp = tmp(:,2:end);
    tmp(:,3) = tmp(:,3)-tmp(:,1); tmp(:,4) = tmp(:,4)-tmp(:,2);          % single
    keep_id = find(proposal_score>=proposal_thr & proposal_pred(:,3)~=0 & proposal_pred(:,4)~=0);
    proposals = double(proposal_pred);
    proposals(:,1) = proposals(:,1)./ratios(2); ...                      % double, ratios = [imgH imgW]./[orgH orgW]

The widths and the compares are single, the division double, and nothing is clipped.  The threshold is compared in
single, as the post-process's cfg holds it; the drivers' -10 and -5 are exact in single, so that is MATLAB's compare.
"""
from __future__ import annotations

import numpy as np


def ratios(net_hw, org_hw) -> tuple[float, float]:
    """ratios = [imgH imgW] ./ [orgH orgW] in double (run_mscnn_detection.m:65)."""
    return float(net_hw[0]) / float(org_hw[0]), float(net_hw[1]) / float(org_hw[1])


def proposals(proposals_score, proposal_thr: float, net_hw, org_hw) -> np.ndarray:
    """One image's rows of proposals_score ([R][6] = img x1 y1 x2 y2 score, float32, as the forward left them;
    an image without proposals has the zero dummy row) -> float64 [k][5] = x y w h score."""
    tmp = np.asarray(proposals_score, dtype=np.float32).reshape(-1, 6)[:, 1:].copy()
    tmp[:, 2] = tmp[:, 2] - tmp[:, 0]
    tmp[:, 3] = tmp[:, 3] - tmp[:, 1]
    with np.errstate(invalid="ignore"):
        keep = (tmp[:, 4] >= np.float32(proposal_thr)) & (tmp[:, 2] != 0) & (tmp[:, 3] != 0)
    p = tmp[keep].astype(np.float64)
    rh, rw = ratios(net_hw, org_hw)
    p[:, 0] = p[:, 0] / rw
    p[:, 2] = p[:, 2] / rw
    p[:, 1] = p[:, 1] / rh
    p[:, 3] = p[:, 3] / rh
    return p


def split_rows(proposals_score, counts) -> list[np.ndarray]:
    """A batch's proposals_score rows cut into images by the per-image row counts."""
    rows = np.asarray(proposals_score).reshape(-1, 6)
    out, start = [], 0
    for c in counts:
        out.append(rows[start:start + int(c)])
        start += int(c)
    return out


def dlmwrite(props, first_index: int = 1) -> bytes:
    """dlmwrite(file, [index x y w h score]) of the float64 rows: ',' delimiter, %.5g, '\\n'."""
    lines = []
    for i, p in enumerate(props):
        for row in np.asarray(p, dtype=np.float64).reshape(-1, 5):
            lines.append(",".join("%.5g" % v for v in [float(first_index + i), *row]) + "\n")
    return "".join(lines).encode()
