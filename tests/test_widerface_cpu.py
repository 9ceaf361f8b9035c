"""The WIDER FACE driver pieces that need no device: the size-bucketed batch plan, the drivers' post-process settings
and the result-file writer (examples/widerface/run_mscnn_detection.m:177-196), against bytes derived by hand from the
MATLAB lines `fprintf(fid, '%s\\n', name)`, `fprintf(fid, '%d\\n', numDets)` and
`fprintf(fid, '%d %d %d %d %f\\n', round(x), round(y), round(w), round(h), prob)`."""
import ctypes as C

import numpy as np
import pytest

from oracle import port


def _wider_sizes(n=60, seed=11):
    """WIDER-like original sizes: widths mostly 1024, heights spread, a few large images above 2048 and 3072."""
    rng = np.random.default_rng(seed)
    sizes = [(int(rng.integers(300, 1800)), 1024) for _ in range(n)]
    sizes += [(2400, 1024), (4000, 3001), (3100, 3100), (683, 1024), (700, 1024), (1024, 768), (3500, 2200)]
    return sizes


def test_plan_batches_cover_group_and_bound():
    from mscnn_b200 import widerface
    sizes = _wider_sizes()
    for max_batch, budget in ((8, widerface.PIXEL_BUDGET), (3, widerface.PIXEL_BUDGET), (8, 2_000_000), (5, 1)):
        plan = widerface.plan_batches(sizes, max_batch=max_batch, pixel_budget=budget)
        flat = [i for _, idx in plan for i in idx]
        assert sorted(flat) == list(range(len(sizes)))                       # every image exactly once
        for (rh, rw), idx in plan:
            assert idx and idx == sorted(idx)
            for i in idx:                                                    # one net size per batch: the driver's
                assert port.widerface_net_size(*sizes[i], 0, 0, 3072) == (rh, rw)
            assert len(idx) <= max_batch
            assert len(idx) == 1 or len(idx) * rh * rw <= budget
        assert widerface.plan_batches(sizes, max_batch=max_batch, pixel_budget=budget) == plan   # deterministic
    plan = widerface.plan_batches(sizes)
    hws = [hw for hw, _ in plan]
    assert len(set(hws)) >= 5 and max(h for h, _ in hws) > 2048                # several sizes, some above 2048
    assert (2400, 1024) in hws                       # max_size 3072: the helper's 2048 default would have scaled it
    areas = [h * w for h, w in hws]
    assert areas == sorted(areas, reverse=True)      # largest net size first


def test_plan_batches_budget_and_lone_large_image():
    from mscnn_b200 import widerface
    sizes = [(768, 1024)] * 11 + [(3072, 3072), (3070, 3080), (768, 1024)]
    plan = widerface.plan_batches(sizes)
    big = [idx for hw, idx in plan if hw == (3072, 3072)]
    assert big == [[11], [12]]                        # 9.4 M pixels each: one per batch under the 8 x 768 x 2560 budget
    small = [idx for hw, idx in plan if hw == (768, 1024)]
    assert small == [list(range(8)), [8, 9, 10, 13]]  # max_batch 8, input order
    # a budget below one image: it still runs, alone
    plan = widerface.plan_batches([(100, 100), (96, 96), (3000, 3000)], pixel_budget=5000)
    assert plan == [((3008, 3008), [2]), ((96, 96), [0]), ((96, 96), [1])]
    # a fixed net size (imgH / imgW set in the driver) puts every image into one group
    plan = widerface.plan_batches([(100, 100), (500, 700), (90, 2000)], img_hw=(512, 512))
    assert plan == [((512, 512), [0, 1, 2])]
    with pytest.raises(ValueError):
        widerface.plan_batches(sizes, max_batch=0)


def test_widerface_detect_cfg_holds_the_driver_constants():
    from mscnn_b200 import net as mnet
    cfg, classes = mnet.widerface_detect_cfg(768, 1024)
    assert (cfg.num_cls, cfg.cls_id) == (2, 2)
    assert list(cfg.bbox_std) == list(np.float32([0.1, 0.1, 0.2, 0.2])) and list(cfg.bbox_mean) == [0.0] * 4
    assert cfg.proposal_thr == -5.0 and cfg.nms_overlap == np.float32(0.3)
    assert cfg.max_rois_per_image >= 3000                                    # BoxOutput max_nms_num of the WIDER nets
    assert (cfg.ratio_h, cfg.ratio_w, cfg.org_h, cfg.org_w) == (1.0, 1.0, 768.0, 1024.0)
    assert classes.num_ids == 1 and classes.cls_ids[0] == 2 and classes.det_thr == np.float32(0.05)
    cfg, _ = mnet.widerface_detect_cfg(672, 1024, org_hw=(683, 1024))
    assert cfg.ratio_h == np.float32(672 / 683) and (cfg.org_h, cfg.org_w) == (683.0, 1024.0)


# ------------------------------------------------------------------------------------------------ result files
ROWS = {
    # round(2.5) = 3, round(-0.5) = -1, round(10.4999) = 10, round(3.5) = 4; prob to six places
    "0_Parade_marchingband_1_20": [[2.5, -0.5, 10.4999, 3.5, 0.123456789],
                                   # -0.4 -> -0 printed as 0; 0.5 -> 1; round(-2.5) = -3; 1000 stays
                                   [-0.4, 0.5, -2.5, 1000.0, 1.0],
                                   [7.49, 0.0, 1.5, 99.5, 0.05]],
    "img.with.dots": [],                                                     # zero detections
    "12_Group_Group_12_Group_Group_12_10.v2": [[319.6, 41.2, 12.5, 14.5, 1 / 3]],
}
EXPECTED = {
    "0_Parade_marchingband_1_20.txt": b"0_Parade_marchingband_1_20\n3\n"
                                      b"3 -1 10 4 0.123457\n"
                                      b"0 1 -3 1000 1.000000\n"
                                      b"7 0 2 100 0.050000\n",
    "img.with.dots.txt": b"img.with.dots\n0\n",
    "12_Group_Group_12_Group_Group_12_10.v2.txt": b"12_Group_Group_12_Group_Group_12_10.v2\n1\n320 41 13 15 0.333333\n",
}


def test_write_results_bytes(tmp_path):
    from mscnn_b200 import widerface
    event = tmp_path / "detections" / "comp" / "0--Parade"          # missing parents are created (mkdir)
    widerface.write_results(event, ROWS)
    assert sorted(p.name for p in event.iterdir()) == sorted(EXPECTED)
    for name, want in EXPECTED.items():
        assert (event / name).read_bytes() == want, name
    widerface.write_results(event, {"img.with.dots": [[1.0, 2.0, 3.0, 4.0, 0.5]]})   # rewrites an existing file
    assert (event / "img.with.dots.txt").read_bytes() == b"img.with.dots\n1\n1 2 3 4 0.500000\n"
    widerface.write_results(tmp_path / "empty_event", {})
    assert (tmp_path / "empty_event").is_dir()


def test_write_results_rejects_bad_arguments_before_touching_the_disk(tmp_path):
    from mscnn_b200 import capi
    L = capi.lib()
    target = tmp_path / "never"

    def call(d=str(target), n=2, names=("a", "b"), dets=None, counts=(1, 0), cap=2):
        dets = np.zeros((2, 2, 5), np.float32) if dets is None else dets
        arr = (C.c_char_p * 2)(*[None if s is None else s.encode() for s in names]) if names is not None else None
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        return L.mscnn_widerface_write_results(None if d is None else d.encode(), n, arr, dets.ctypes.data,
                                               cnt.ctypes.data, cap)

    nan = np.zeros((2, 2, 5), np.float32)
    nan[0, 0, 2] = np.nan
    inf = np.zeros((2, 2, 5), np.float32)
    inf[0, 0, 4] = np.inf
    for kw in (dict(d=None), dict(d=""), dict(n=-1), dict(cap=0), dict(names=None), dict(names=("a", None)),
               dict(names=("", "b")), dict(names=("a", "../b")), dict(counts=(3, 0)), dict(counts=(-1, 0)),
               dict(dets=nan), dict(dets=inf)):
        assert call(**kw) == capi.ERR_INVALID, kw
        assert not target.exists(), kw
    nan[0, 1, 2] = np.nan                            # beyond the kept rows of image 0: never read
    nan[0, 0, 2] = 0.0
    assert call(dets=nan) == capi.OK
    assert (target / "a.txt").read_bytes() == b"a\n1\n0 0 0 0 0.000000\n"
    assert (target / "b.txt").read_bytes() == b"b\n0\n"
