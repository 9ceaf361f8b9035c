"""Inputs for BoxOutput and the final-detection post-process whose decoded boxes are the same bits on the device and in
oracle.port, each built to sit on one discrete edge: an IoU exactly on the threshold, a greedy chain across the NMS
kernels' 64-box blocks, a run of equal scores across the top-K cut, counts around K and the block sizes, empty images
in a batch, non-finite map values.

Exact geometry:
* BoxOutput: power-of-two fields, anchor rates 8 / 16, x/y deltas that are multiples of 1 / field and width/height
  deltas of 0 (exp(0) = 1), so every centre and corner is an integer and no rounding happens anywhere.  A case that
  needs another exp argument checks that glibc's expf and the once-rounded fp64 exp agree on it (exp_unambiguous).
* Scores: background channel 0, one class channel = the wanted score, so fg is exactly that value (-0.0 stays -0.0).
* Post-process: integer boxes, ratios 1, zero box deltas; logits only where exp_unambiguous holds.

Each case carries `claims`, checked with the oracle alone by test_box_edges_cpu.py, so that a builder that loses its
edge fails there; test_box_edges_gpu.py compares the device with the oracle bit for bit on the same cases.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math
from dataclasses import dataclass, field

import numpy as np

from oracle import port

F32 = np.float32
_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.expf.restype = ctypes.c_float
_libm.expf.argtypes = [ctypes.c_float]
_libm.logf.restype = ctypes.c_float
_libm.logf.argtypes = [ctypes.c_float]


def exp_unambiguous(v) -> bool:
    """glibc expf(v) equals float32(exp(float64(v))), and exp(v) is not within 2^-40 (relative) of a midpoint between
    two floats, so any exp that is faithful in fp64 rounds to the same float."""
    v = float(F32(v))
    e = math.exp(v)
    f = F32(e)
    if F32(_libm.expf(v)) != f:
        return False
    lo = float(np.nextafter(f, F32(-np.inf)))
    hi = float(np.nextafter(f, F32(np.inf)))
    mids = [(lo + float(f)) / 2, (float(f) + hi) / 2]
    return all(abs(e - m) > 2.0 ** -40 * e for m in mids)


def logf(v) -> float:
    return float(_libm.logf(float(v)))


# ------------------------------------------------------------------------------------------------------ BoxOutput
@dataclass
class Scale:
    h: int          # map rows
    w: int          # map columns
    field: int      # anchor box size (power of two)
    rate: int       # anchor stride in image pixels


@dataclass
class BoxCase:
    name: str
    edge: str
    maps: list
    scales: list
    cfg: dict
    claims: dict = field(default_factory=dict)

    @property
    def n(self) -> int:
        return self.maps[0].shape[0]

    def oracle_args(self, **over):
        c = dict(self.cfg, **over)
        return dict(field_w=[s.field for s in self.scales], field_h=[s.field for s in self.scales],
                    downsample_rate=[s.rate for s in self.scales], fg_thr=c["fg_thr"], iou_thr=c["iou_thr"],
                    nms_type=c["nms_type"], field_whr=c["field_whr"], field_xyr=c["field_xyr"],
                    min_size=c["min_size"], max_nms_num=c["max_nms_num"], max_post_nms_num=c["max_post_nms_num"])

    def oracle(self, **over):
        """port.box_output on the case, with cfg entries replaced by `over`."""
        return port.box_output(self.maps, **self.oracle_args(**over))


def box_cfg(**kw) -> dict:
    c = dict(fg_thr=-100.0, iou_thr=0.6, nms_type="IOU", field_whr=2.0, field_xyr=2.0, min_size=4.0,
             max_nms_num=300, max_post_nms_num=0)
    c.update(kw)
    return c


class Canvas:
    """N images of score/delta maps over `scales`, `channels` = background + classes + 4 deltas.  Every anchor starts
    rejected (background +inf, classes -inf: fg = -inf); place() makes one anchor decode to a chosen box and score."""

    def __init__(self, n, scales, channels=6, field_xyr=2.0):
        self.scales = scales
        self.ch = channels
        self.maps = []
        for s in scales:
            m = np.zeros((n, channels, s.h, s.w), F32)
            m[:, 0] = np.inf
            m[:, 1:channels - 4] = -np.inf
            self.maps.append(m)
        self.reach = [int(s.field / field_xyr) for s in scales]   # max |dx * field| in pixels
        self.base = np.cumsum([0] + [s.h * s.w for s in scales])[:-1]

    def img_w(self, j):
        return self.scales[j].w * self.scales[j].rate

    def img_h(self, j):
        return self.scales[j].h * self.scales[j].rate

    def free(self, n, j, h, w) -> bool:
        return self.maps[j][n, 0, h, w] == np.inf

    def set_anchor(self, n, j, h, w, x, y, score):
        """Anchor (h, w) of scale j decodes to the box [x, y, field, field] with fg = score."""
        s = self.scales[j]
        cx, cy = x + s.field // 2, y + s.field // 2
        ox, oy = cx - (2 * w + 1) * s.rate // 2, cy - (2 * h + 1) * s.rate // 2
        assert abs(ox) <= self.reach[j] and abs(oy) <= self.reach[j], (ox, oy)
        assert 0 <= x and x + s.field <= self.img_w(j) and 0 <= y and y + s.field <= self.img_h(j), (x, y)
        m = self.maps[j]
        m[n, 0, h, w] = 0.0
        m[n, 1, h, w] = F32(score)
        m[n, self.ch - 4, h, w] = F32(ox / s.field)
        m[n, self.ch - 3, h, w] = F32(oy / s.field)
        m[n, self.ch - 2, h, w] = 0.0
        m[n, self.ch - 1, h, w] = 0.0
        return int(self.base[j] + h * s.w + w)

    def place(self, n, j, x, y, score) -> int:
        """The box [x, y, field, field] of scale j on the nearest free anchor within reach; returns the anchor index."""
        s = self.scales[j]
        cx, cy = x + s.field // 2, y + s.field // 2
        w0, h0 = int(round(cx / s.rate - 0.5)), int(round(cy / s.rate - 0.5))
        r = self.reach[j] // s.rate
        offs = sorted(((dh, dw) for dh in range(-r, r + 1) for dw in range(-r, r + 1)), key=lambda t: t[0] ** 2 + t[1] ** 2)
        for dh, dw in offs:
            h, w = h0 + dh, w0 + dw
            if not (0 <= h < s.h and 0 <= w < s.w) or not self.free(n, j, h, w):
                continue
            if abs(cx - (2 * w + 1) * s.rate // 2) > self.reach[j] or abs(cy - (2 * h + 1) * s.rate // 2) > self.reach[j]:
                continue
            return self.set_anchor(n, j, h, w, x, y, score)
        raise ValueError(f"no free anchor for box ({x}, {y}) on scale {j}")

    def case(self, name, edge, cfg, claims=None) -> BoxCase:
        return BoxCase(name, edge, self.maps, self.scales, cfg, claims or {})


TWO_SCALES = [Scale(48, 96, 64, 8), Scale(24, 48, 128, 16)]     # both 768 x 384 pixels


def threshold_tie_cases() -> list[BoxCase]:
    """Pairs whose fp32 BoxIOU is exactly iou_thr (kept: the test is a strict >), beside pairs one pixel nearer
    (suppressed) and farther (kept), on both scales; the same maps at the threshold and one float either side."""
    out = []
    for mode in ("IOU", "IOMU", "IOFU"):
        for step in (-1, 0, 1):
            cv = Canvas(1, TWO_SCALES)
            score = 1000.0
            ties, near = [], []
            # scale 0: 64 x 64 boxes 16 px apart: IOU 3072 / 5120 = float32(0.6); IOMU / IOFU 3072 / 4096 = 0.75
            for k, (x, y) in enumerate([(8, 8), (104, 8), (200, 8), (296, 8), (8, 96), (104, 96)]):
                d = (16, 15, 17)[k % 3]
                a, b = (x, y, 64, 64), (x + d, y, 64, 64)
                cv.place(0, 0, x, y, score)
                cv.place(0, 0, x + d, y, score - 1)
                score -= 2
                (ties if d == 16 else near).append((0, a, b))
            # scale 1: two 128 boxes 32 apart (IOU 12288 / 20480 = float32(0.6), IOMU / IOFU 0.75); a 64 box ranked
            # first with 48 of its 64 columns inside a 128 box (IOMU / IOFU 3072 / 4096 = 0.75)
            cv.place(0, 1, 400, 16, score)
            cv.place(0, 1, 432, 16, score - 1)
            ties.append((0, (400, 16, 128, 128), (432, 16, 128, 128)))
            cv.place(0, 0, 400, 200, score - 2)
            cv.place(0, 1, 416, 168, score - 3)
            if mode != "IOU":
                ties.append((0, (400, 200, 64, 64), (416, 168, 128, 128)))
            t = F32(port.box_iou(*ties[0][1:], mode))
            thr = t if step == 0 else np.nextafter(t, F32(-step * np.inf))
            where = {-1: "iou_thr one float above the tie", 0: "iou_thr exactly the tie",
                     1: "iou_thr one float below the tie"}[step]
            cfg = box_cfg(nms_type=mode, iou_thr=float(thr), max_nms_num=64)
            out.append(cv.case(f"iou_tie_{mode}_{['thr_above', 'thr_at', 'thr_below'][step + 1]}",
                               f"{mode} pairs at {float(t)!r}, {where}: tie pairs {'kept' if step <= 0 else 'suppressed'}",
                               cfg, dict(tie_pairs=ties, tie_value=float(t), tie_kept=step <= 0)))
    return out


def _chain_rows(cv, n, y0, ranks, score_of, rows_per, x0=8, pitch=15):
    """Greedy chains: rows of boxes `pitch` px apart (IoU(15) = 0.62 > 0.6, IoU(30) = 0.36), rank order along the
    row, so the greedy scan keeps every other box of a row.  Rows are 80 px apart and do not interact."""
    for i, r in enumerate(ranks):
        row, col = divmod(i, rows_per)
        cv.place(n, 0, x0 + pitch * col, y0 + 80 * row, score_of(r))


def greedy_chain_cases() -> list[BoxCase]:
    out = []
    # a lone box at rank 0, then chains of 81 boxes: the rows span ranks 1-81, 82-162, 163-243, 244-324, ...: block 1
    # starts with its first box suppressed by the last kept box of block 0, block 2 passes through a chain, and so on
    for total, k in ((330, 330), (8192, 8192)):
        rows_per = 81
        nrows = (total - 1 + rows_per - 1) // rows_per
        cv = Canvas(1, [Scale((80 * (nrows + 1) + 16) // 8 + 1, 160, 64, 8)])
        cv.place(0, 0, 8, 8 + 80 * nrows, 10000.0)
        _chain_rows(cv, 0, 8, list(range(1, total)), lambda r: 10000.0 - r, rows_per)
        out.append(cv.case(f"greedy_chain_{total}", f"greedy chains across the 64-box blocks, {(k + 63) // 64} blocks",
                           box_cfg(max_nms_num=k), dict(chain_edges=True)))
    return out


def _grid_positions(count, x0, y0, cols, pitch=32):
    return [(x0 + pitch * (i % cols), y0 + pitch * (i // cols)) for i in range(count)]


def k_tie_cases() -> list[BoxCase]:
    """A run of equal scores straddling position K (the anchor index decides), spread over both scales, with boxes
    32 px apart (IoU <= 1/3: no suppression at iou_thr 0.6) so the cut at K shows in the output."""
    out = []
    rng = np.random.default_rng(2024)
    for k, run_val, above, below in [(1, 2.5, 0, 40), (63, -2.5, 40, 60), (64, 3.0, 30, 30), (65, 0.0, 20, 40),
                                     (64, "pm0", 33, 20), (65, "pm0", 0, 30), (2049, "pm0", 1500, 300),
                                     (64, np.inf, 0, 20), (2049, -1.0, 1900, 100)]:
        run = (k + 40) - above if above < k else 40
        total = above + run + below
        cols0 = 22
        n0 = (2 * total) // 3
        rows0 = (n0 + cols0 - 1) // cols0
        h0 = (32 * rows0 + 64 + 8) // 8 + 1
        n1 = total - n0
        cols1 = 4
        rows1 = (n1 + cols1 - 1) // cols1
        h1 = (8 * h0 + 160 * rows1 + 128 + 16) // 16 + 1
        scales = [Scale(h0, 96, 64, 8), Scale(h1, 48, 128, 16)]
        cv = Canvas(1, scales)
        pos = [(0, x, y) for x, y in _grid_positions(n0, 8, 8, cols0)]
        pos += [(1, x, y) for x, y in _grid_positions(n1, 8, 8 * h0 + 8, cols1, pitch=160)]
        order = rng.permutation(total)          # which position gets which rank: index order != rank order
        scores = [100.0 + above - i for i in range(above)] + [0.0 if run_val == "pm0" else run_val] * run \
            + [-50.0 - i for i in range(below)]
        idx = [cv.place(0, *pos[p], s) for p, s in zip(order, scores)]
        idx_of = dict(zip(order, idx))
        if run_val == "pm0":
            # the run's larger anchor indices get -0.0: the reference ranks them first (-0 == +0, then the larger
            # index); a key that orders +0 above -0 would cut the other part of the run
            run_pos = sorted(order[above:above + run], key=lambda p: idx_of[p])
            for p in run_pos[len(run_pos) // 3:]:
                j = pos[p][0]
                a = idx_of[p] - int(cv.base[j])
                cv.maps[j][0, 1, a // scales[j].w, a % scales[j].w] = F32(-0.0)
        label = {"pm0": "pm0", np.inf: "inf"}.get(run_val, str(run_val))
        fg_thr = -1e4
        out.append(cv.case(f"k_tie_K{k}_{label}_above{above}", f"K = {k} inside a run of {run} scores {label}",
                           box_cfg(max_nms_num=k, fg_thr=fg_thr),
                           dict(k_tie=k, signed_zero=run_val == "pm0", valid=[total])))
    return out


def _random_canvas(n, valid_per_image, seed, scales=None):
    """Random integer geometry on every chosen anchor (x/y deltas in multiples of 1/field within reach, boxes of 64
    and 128 px that overlap heavily) and scores on a 0.5 grid (many ties)."""
    if scales is None:
        # the smallest canvas that holds the anchors, so that small counts overlap as densely as large ones
        for a, b in ((16, 12), (64, 32), (96, 48), (128, 64)):
            scales = [Scale(a, a, 64, 8), Scale(b, b, 128, 16)]
            if a * a + b * b >= max(valid_per_image):
                break
    cv = Canvas(n, scales)
    rng = np.random.default_rng(seed)
    total = sum(s.h * s.w for s in scales)
    for i, v in enumerate(valid_per_image):
        assert v <= total
        for a in rng.choice(total, size=v, replace=False):
            j = int(np.searchsorted(cv.base, a, side="right") - 1)
            s = scales[j]
            h, w = divmod(int(a - cv.base[j]), s.w)
            r = cv.reach[j]
            cx = (2 * w + 1) * s.rate // 2 + int(rng.integers(-r, r + 1))
            cy = (2 * h + 1) * s.rate // 2 + int(rng.integers(-r, r + 1))
            x = min(max(cx - s.field // 2, 0), cv.img_w(j) - s.field)
            y = min(max(cy - s.field // 2, 0), cv.img_h(j) - s.field)
            cv.set_anchor(i, j, h, w, x, y, float(rng.integers(-16, 17)) * 0.5)
    return cv


COUNT_KS = (1, 63, 64, 65, 2048, 2049, 4097, 8192)


def count_cases() -> list[BoxCase]:
    """max_nms_num K against valid-anchor counts 0, K - 1, K, K + 1 and 2K + 37, with dense overlapping boxes."""
    out = []
    for k in COUNT_KS:
        for v in sorted({0, k - 1, k, k + 1, 2 * k + 37}):
            cv = _random_canvas(1, [v], seed=k * 7 + v)
            out.append(cv.case(f"count_K{k}_valid{v}", f"K = {k}, {v} valid anchors",
                               box_cfg(max_nms_num=k), dict(valid=[v], suppresses=min(v, k) > 2)))
    return out


def post_nms_cases() -> list[BoxCase]:
    """max_post_nms_num 63, 64, 65, 128 against images that keep 64 and 130 boxes: every grid box has a lower-scored
    partner 8 px to its right (IoU 0.78, suppressed)."""
    out = []
    for mp in (63, 64, 65, 128):
        cv = Canvas(2, [Scale(128, 112, 64, 8)])
        for n, kept in enumerate((64, 130)):
            for i, (x, y) in enumerate(_grid_positions(kept, 8, 8, 11, pitch=80)):
                cv.place(n, 0, x, y, 500.0 - i)
                cv.place(n, 0, x + 8, y, 100.0 - i)
        out.append(cv.case(f"post_nms_{mp}", f"max_post_nms_num {mp} against 64 and 130 kept",
                           box_cfg(max_nms_num=512, max_post_nms_num=mp), dict(kept_uncapped=[64, 130])))
    return out


def batch_cases() -> list[BoxCase]:
    """N = 1 and 3 with an empty image first, in the middle, last, and everywhere (the dummy row)."""
    out = []
    for counts in ([0], [700], [0, 500, 900], [400, 0, 650], [800, 300, 0], [0, 0, 0]):
        cv = _random_canvas(len(counts), counts, seed=sum(counts) + len(counts))
        out.append(cv.case("batch_" + "_".join(map(str, counts)), f"per-image valid counts {counts}",
                           box_cfg(max_nms_num=300), dict(valid=counts)))
    return out


def nonfinite_cases() -> list[BoxCase]:
    """Two classes: NaN in a class channel (the other class decides), NaN in the background (anchor rejected), NaN and
    +-inf in the deltas (clamped to the delta limits; exp of log(2) and log(1/2) checked unambiguous)."""
    assert exp_unambiguous(logf(2.0)) and exp_unambiguous(logf(F32(1.0) / F32(2.0)))
    cv = Canvas(1, [Scale(48, 96, 64, 8)], channels=7)
    m = cv.maps[0]
    for i, (x, y) in enumerate(_grid_positions(120, 40, 40, 15, pitch=40)):
        a = cv.place(0, 0, x, y, 50.0 - i)
        h, w = divmod(a, 96)
        kind = i % 8
        if kind == 1:
            m[0, 1, h, w], m[0, 2, h, w] = np.nan, F32(20.0 - i)          # class 1 NaN: class 2 is the score
        elif kind == 2:
            m[0, 0, h, w] = np.nan                                        # background NaN: rejected
        elif kind == 3:
            m[0, 3, h, w] = np.nan                                        # dx NaN -> min_xyr
        elif kind == 4:
            m[0, 5, h, w] = np.nan                                        # dw NaN -> min_whr
        elif kind == 5:
            m[0, 6, h, w] = np.inf                                        # dh +inf -> max_whr
        elif kind == 6:
            m[0, 4, h, w] = -np.inf                                       # dy -inf -> min_xyr
        elif kind == 7:
            m[0, 1, h, w], m[0, 2, h, w] = F32(30.0 - i), np.nan          # class 2 NaN: class 1 is the score
    return [cv.case("nonfinite", "NaN / inf in class, background and delta channels", box_cfg(max_nms_num=128),
                    dict(valid=[120 - 15]))]


def box_cases() -> list[BoxCase]:
    return (threshold_tie_cases() + greedy_chain_cases() + k_tie_cases() + count_cases() + post_nms_cases()
            + batch_cases() + nonfinite_cases())


# ------------------------------------------------------------------------------------------- final-detection post-process
@dataclass
class DetCase:
    name: str
    edge: str
    cascade: bool
    prop: np.ndarray        # [R, 6] proposals_score (MS-CNN) or [R, 5] proposals (cascade)
    cls: np.ndarray         # [R, num_cls] logits (MS-CNN) or probabilities (cascade)
    bbox: np.ndarray        # [R, 4 num_cls] deltas (MS-CNN) or [R, 5] decoded boxes (cascade)
    counts: list            # rows per image
    max_rois: int
    cls_ids: list
    overlap: float = 0.5
    det_thr: float = -1.0
    org_hw: tuple = (2048.0, 4096.0)
    claims: dict = field(default_factory=dict)

    @property
    def n(self) -> int:
        return len(self.counts)

    @property
    def num_cls(self) -> int:
        return self.cls.shape[1]

    def num_out(self) -> np.ndarray:
        r = int(sum(self.counts))
        return np.array([max(r, 1), r] + list(self.counts), dtype=np.int32)

    def oracle(self, image, cls_id, overlap=None, det_thr=None) -> np.ndarray:
        """Final detections [K, 5] of one image and class by the restated MATLAB post-process."""
        s = int(sum(self.counts[:image]))
        sl = slice(s, s + self.counts[image])
        ov = self.overlap if overlap is None else overlap
        if self.cascade:
            d = port.cascade_detect_postprocess(self.prop[sl], self.cls[sl], self.bbox[sl], cls_id=cls_id, overlap=ov,
                                                org_hw=self.org_hw)
        else:
            d = port.detect_postprocess(self.prop[sl], self.cls[sl], self.bbox[sl], cls_id=cls_id, overlap=ov,
                                        org_hw=self.org_hw)
        thr = self.det_thr if det_thr is None else det_thr
        return d if thr <= 0 else d[d[:, 4] >= F32(thr)]


def _cascade_rows(boxes, probs, img, num_cls=3, cls_col=1):
    """Cascade blobs for integer boxes (x, y, w, h) in the MATLAB +1 convention: x2 = x + w - 1."""
    b = np.asarray(boxes, np.float64).reshape(-1, 4)
    r = len(b)
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 0] + b[:, 2] - 1, b[:, 1] + b[:, 3] - 1
    prop = np.stack([np.full(r, img), x1, y1, x2, y2], 1).astype(F32)
    out = prop.copy()
    cls = np.full((r, num_cls), F32(0.125), F32)
    cls[:, cls_col] = np.asarray(probs, F32)
    return prop, cls, out


def _concat(parts):
    return [np.concatenate([p[k] for p in parts]) if parts else None for k in range(3)]


def bbnms_overlap(a, b) -> float:
    """bbNms's 'union' overlap of two [x y w h] boxes in double (bbNms.m:112-126)."""
    a, b = [float(v) for v in a], [float(v) for v in b]
    iw = min(a[0] + a[2], b[0] + b[2]) - max(a[0], b[0])
    ih = min(a[1] + a[3], b[1] + b[3]) - max(a[1], b[1])
    if iw <= 0 or ih <= 0:
        return 0.0
    o = iw * ih
    return o / (a[2] * a[3] + b[2] * b[3] - o)


def cascade_tie_cases() -> list[BoxCase]:
    """30-wide boxes 10 apart overlap exactly 0.5 = nms_overlap in double (kept: bbNms tests o > overlap), beside
    pairs 9 apart (suppressed) and 11 apart (kept); horizontal and vertical pairs."""
    out = []
    for step in (-1, 0, 1):
        boxes, probs, ties = [], [], []
        p = 0.9
        for k in range(30):
            x, y = 20 + 100 * (k % 10), 20 + 100 * (k // 10)
            d = (10, 9, 11)[k % 3]
            e = 30 if k % 2 else 40      # the other extent: the overlap (30 - d) / (30 + d) does not depend on it
            a, b = ((x, y, 30, e), (x + d, y, 30, e)) if k % 4 < 2 else ((x, y, e, 30), (x, y + d, e, 30))
            boxes += [a, b]
            probs += [p, p - 0.001]
            p -= 0.002
            if d == 10:
                ties.append((0, a, b))
        ov = 0.5 if step == 0 else float(np.nextafter(F32(0.5), F32(step * np.inf)))
        prop, cls, bbox = _cascade_rows(boxes, probs, 0)
        out.append(DetCase(f"bbnms_tie_{['below', 'at', 'above'][step + 1]}",
                           "bbNms overlap exactly 0.5, nms_overlap " + ["one float below", "0.5", "one float above"][step + 1],
                           True, prop, cls, bbox, [len(boxes)], 64, [2], overlap=ov,
                           claims=dict(tie_pairs=ties, tie_kept=step >= 0, tie_value=0.5)))
    return out


def cascade_order_cases() -> list[DetCase]:
    """Equal probabilities across the 64-row blocks (MATLAB's stable sort: the lower row first), +0 and -0 mixed in
    one run, disjoint boxes so the order is the output order; three images with the empty one in the middle."""
    rng = np.random.default_rng(77)
    parts, counts = [], []
    for img, r in enumerate((300, 0, 200)):
        pos = [(10 + 40 * (i % 40), 10 + 40 * (i // 40), 30, 30) for i in range(r)]
        vals = np.array([0.75, 0.5, 0.5, 0.25, 0.0, -0.0, 0.0], F32)
        probs = vals[rng.integers(0, len(vals), r)]
        probs[:70] = F32(0.5)
        if r:
            probs[100:140] = F32(-0.0)
            probs[140:180] = F32(0.0)
        parts.append(_cascade_rows(pos, probs, img))
        counts.append(r)
    prop, cls, bbox = _concat(parts)
    return [DetCase("prob_ties_blocks", "equal probabilities across 64-row blocks, +0 and -0 in one run", True,
                    prop, cls, bbox, counts, 512, [2], claims=dict(prob_tie_edges=True, signed_zero=True))]


def cascade_count_cases() -> list[DetCase]:
    """Per-image row counts at max_rois_per_image 64, 65, 2048, 8192: random integer boxes that overlap (NMS on every
    block), probabilities on a coarse grid (ties)."""
    out = []
    for cap in (64, 65, 2048, 8192):
        rng = np.random.default_rng(cap)
        parts, counts = [], []
        for img, r in enumerate((cap, cap - 1)):
            side = int(math.sqrt(r) * 24) + 64
            x = rng.integers(0, side, r)
            y = rng.integers(0, side, r)
            w = rng.integers(20, 60, r)
            h = rng.integers(20, 60, r)
            probs = rng.integers(0, 9, r).astype(F32) / F32(8)
            parts.append(_cascade_rows(np.stack([x, y, w, h], 1), probs, img))
            counts.append(r)
        prop, cls, bbox = _concat(parts)
        out.append(DetCase(f"cascade_count_{cap}", f"{cap} and {cap - 1} rows at max_rois_per_image {cap}", True,
                           prop, cls, bbox, counts, cap, [2, 3], claims=dict(rows=counts)))
    return out


LOGITS = [0.0, 0.5, -0.25, 1.0, -1.5, 2.0]


def mscnn_cases() -> list[DetCase]:
    """MS-CNN path: integer proposals, zero box deltas (exp(0) = 1), logit rows repeated from a few patterns (equal
    probabilities across blocks), proposal scores on both sides of proposal_thr; a detection threshold equal to one
    of the tied probabilities."""
    assert all(exp_unambiguous(v) for v in LOGITS)
    out = []
    num_cls = 4
    for cap, rows in ((64, (64, 0, 40)), (65, (65, 65, 0)), (2048, (0, 2048, 1500))):
        rng = np.random.default_rng(cap + 1)
        pats = np.array([rng.choice(LOGITS, num_cls) for _ in range(5)], F32)
        props, clss, counts = [], [], []
        for img, r in enumerate(rows):
            side = int(math.sqrt(max(r, 1)) * 30) + 64
            x = rng.integers(0, side, r)
            y = rng.integers(0, side, r)
            w = rng.integers(10, 70, r)
            h = rng.integers(10, 70, r)
            sc = rng.integers(-12, 4, r).astype(F32)
            props.append(np.stack([np.full(r, img), x, y, x + w, y + h, sc], 1).astype(F32))
            clss.append(pats[rng.integers(0, len(pats), r)])
            counts.append(r)
        prop, cls = np.concatenate(props), np.concatenate(clss)
        bbox = np.zeros((len(prop), 4 * num_cls), F32)
        e = np.exp(pats.astype(np.float64)).astype(F32)
        s = np.zeros(len(pats), F32)
        for k in range(num_cls):
            s = (s + e[:, k]).astype(F32)
        thr = float((e[:, 1] / s).astype(F32)[0])
        out.append(DetCase(f"mscnn_rows_{cap}", f"MS-CNN rows {rows}, repeated logit rows, max_rois_per_image {cap}",
                           False, prop, cls, bbox, counts, cap, [2, 4], det_thr=-1.0,
                           claims=dict(rows=counts, prob_ties=True)))
        out.append(DetCase(f"mscnn_rows_{cap}_det_thr", f"as mscnn_rows_{cap}, det_thr = a tied probability of class 2",
                           False, prop, cls, bbox, counts, cap, [2, 4], det_thr=thr,
                           claims=dict(rows=counts, det_thr_hit=True)))
    return out


def det_cases() -> list[DetCase]:
    return cascade_tie_cases() + cascade_order_cases() + cascade_count_cases() + mscnn_cases()
