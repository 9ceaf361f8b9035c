"""The fixed-size driver specs, their result files and gray frames, host side (no GPU).

(a) Every field of the five specs (mscnn_b200/drivers.py) is pinned to what its .m file sets.
(b) write_results writes, byte for byte, the dlmwrite rows ([index x y w h p], ',' and %.5g) of the drivers, for
    seeded detections with empty images, and with CityPersons' index running across two groups of frames.
(c) A gray frame through the CPU restatement of the pre-processing (oracle/port.py) equals its repmat to three channels,
    and the C ABI rejects 2- and 4-channel frames before any CUDA call."""
import ctypes as C

import numpy as np
import pytest


def test_specs_match_the_driver_scripts():
    from mscnn_b200 import drivers as D
    k = D.KITTI_CAR
    assert k.script == "examples/kitti_car/run_mscnn_detection.m"
    assert k.net_hw == (768, 2560) and k.num_cls == 5 and k.cls_ids == (2,) and not k.cascade
    assert k.obj_names == ("bg", "car", "van", "truck", "tram")
    assert k.blobs == ("proposals_score", "cls_pred", "bbox_pred")
    assert k.bbox_stds == (0.1, 0.1, 0.2, 0.2) and k.proposal_thr == -10.0 and k.nms_overlap == 0.5
    assert k.det_thr == -1.0 and k.result_files == ("{comp_id}_car.txt",) and not k.index_across_groups

    p = D.KITTI_PED_CYC
    assert p.script == "examples/kitti_ped_cyc/run_mscnn_detection.m"
    assert p.net_hw == (768, 2560) and p.num_cls == 3 and p.cls_ids == (2, 3) and p.obj_names == ("bg", "ped", "cyc")
    assert p.bbox_stds == (0.1, 0.1, 0.2, 0.2) and p.proposal_thr == -10.0 and p.nms_overlap == 0.5
    assert p.result_files == ("{comp_id}_ped.txt", "{comp_id}_cyc.txt") and p.blobs == k.blobs

    c = D.CALTECH
    assert c.script == "examples/caltech/run_mscnn_detection.m"
    assert c.net_hw == (720, 960) and c.num_cls == 2 and c.cls_ids == (2,) and c.obj_names == ("bg", "ped")
    assert c.bbox_stds is None                                  # do_bb_norm = 0 (:41-48)
    assert c.proposal_thr == -10.0 and c.nms_overlap == 0.5 and c.result_files == ("{comp_id}_ped.txt",)

    kc = D.KITTI_CAR_CASCADE
    assert kc.script == "examples/kitti_car/run_cascademscnn.m"
    assert kc.net_hw == (576, 1920) and kc.num_cls == 5 and kc.cls_ids == (2,) and kc.cascade
    assert kc.blobs == ("proposals_3rd", "cls_prob_3rd", "output_bbox_3rd")
    assert kc.det_thr == -1.0 and kc.nms_overlap == 0.5 and kc.proposal_thr is None
    assert kc.result_files == ("{comp_id}_car_3rd_results.txt",) and not kc.index_across_groups

    cp = D.CITYPERSONS
    assert cp.script == "examples/citypersons/run_cascademscnn.m"
    assert cp.net_hw == (1344, 2688) and cp.num_cls == 2 and cp.cls_ids == (2,) and cp.cascade
    assert cp.blobs == ("proposals_3rd", "cls_prob_3rd_avg", "output_bbox_3rd")
    assert cp.det_thr == -1.0 and cp.nms_overlap == 0.5 and cp.obj_names is None
    assert cp.result_files == ("{comp_id}_3rd_avg_results.txt",) and cp.index_across_groups

    for s in D.SPECS.values():
        if s.cascade:                       # imgH = round(imgH/32)*32 leaves the cascade drivers' sizes as they are
            assert s.net_hw[0] % 32 == 0 and s.net_hw[1] % 32 == 0
        assert {"net_hw", "cls_ids", "blobs", "det_thr", "result_files", "index"} <= set(s.source), s.script
        if s.obj_names is not None:         # the file names come from obj_names{id}
            assert all(s.obj_names[i - 1] in f for i, f in zip(s.cls_ids, s.result_files))


def test_detect_cfg_says_what_the_specs_say():
    from mscnn_b200 import drivers as D, net as mnet
    cfg, k = D.KITTI_CAR.detect_cfg()
    ref = mnet.kitti_detect_cfg(768, 2560)
    assert bytes(cfg) == bytes(ref)
    assert (k.num_ids, k.cls_ids[0], k.det_thr) == (1, 2, -1.0)
    cfg, k = D.KITTI_PED_CYC.detect_cfg((192, 640))
    ref, ref_k = mnet.kitti_ped_cyc_detect_cfg(192, 640)
    assert bytes(cfg) == bytes(ref) and bytes(k) == bytes(ref_k)
    cfg, _ = D.CALTECH.detect_cfg()
    assert list(cfg.bbox_std) == [1.0] * 4 and list(cfg.bbox_mean) == [0.0] * 4 and cfg.num_cls == 2
    assert cfg.proposal_thr == -10.0 and (cfg.ratio_h, cfg.ratio_w) == (1.0, 1.0)
    for s in (D.KITTI_CAR_CASCADE, D.CITYPERSONS):
        cfg, k = s.detect_cfg()
        assert cfg.num_cls == s.num_cls and abs(cfg.nms_overlap - 0.5) < 1e-7 and k.det_thr == -1.0


def _seeded_results(n_images, n_cls, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_images):
        per = []
        for c in range(n_cls):
            k = 0 if (i + c) % 3 == 1 else int(rng.integers(1, 6))     # some images have no detections
            xywh = rng.uniform(0, 1200, size=(k, 4)) * rng.choice([1.0, 1e-3, 12.5], size=(k, 1))
            p = rng.uniform(0, 1, size=(k, 1))
            per.append(np.hstack([xywh, p]).astype(np.float32))
        out.append(per)
    return out


def _dlmwrite(results, cls, first_index):
    """dlmwrite(file, [index x y w h p]) of MATLAB's defaults: ',' delimiter, %.5g, '\\n'."""
    lines = []
    for i, r in enumerate(results):
        for row in r[cls]:
            lines.append(",".join("%.5g" % float(v) for v in [first_index + i, *row]) + "\n")
    return "".join(lines).encode()


@pytest.mark.parametrize("name", ["kitti_car", "kitti_ped_cyc", "caltech", "kitti_car_cascade"])
def test_result_files_are_the_drivers_dlmwrite(tmp_path, name):
    from mscnn_b200 import drivers as D
    spec = D.SPECS[name]
    res = _seeded_results(11, len(spec.cls_ids), seed=len(name))
    paths = D.write_results(tmp_path / "detections", spec, "comp_x", res)
    assert [p.name for p in paths] == [f.format(comp_id="comp_x") for f in spec.result_files]
    for c, p in enumerate(paths):
        assert p.read_bytes() == _dlmwrite(res, c, 1), (name, c)
    # a later part of the list: the index starts where the caller says
    paths = D.write_results(tmp_path / "part", spec, "comp_x", res[4:], first_index=5)
    for c, p in enumerate(paths):
        assert p.read_bytes() == _dlmwrite(res[4:], c, 5)
        full = _dlmwrite(res, c, 1).decode().splitlines(keepends=True)
        assert p.read_text() == "".join(l for l in full if int(l.split(",")[0]) >= 5)


def test_citypersons_index_runs_across_groups(tmp_path):
    from mscnn_b200 import drivers as D
    spec = D.CITYPERSONS
    city_a, city_b = _seeded_results(5, 1, seed=3), _seeded_results(7, 1, seed=4)
    paths = D.write_results(tmp_path, spec, "mscnn_8s_1344_2x", [city_a, city_b], groups=True)
    assert [p.name for p in paths] == ["mscnn_8s_1344_2x_3rd_avg_results.txt"]
    assert paths[0].read_bytes() == _dlmwrite(city_a + city_b, 0, 1)
    idx = [int(l.split(",")[0]) for l in paths[0].read_text().splitlines()]
    assert idx == sorted(idx) and max(idx) > 5                    # city b's images are numbered 6..12
    with pytest.raises(ValueError):
        D.write_results(tmp_path, D.KITTI_PED_CYC, "x", _seeded_results(2, 1, seed=0))


def test_all_empty_writes_empty_files(tmp_path):
    from mscnn_b200 import drivers as D
    res = [[np.zeros((0, 5), np.float32), np.zeros((0, 5), np.float32)] for _ in range(3)]
    for p in D.write_results(tmp_path, D.KITTI_PED_CYC, "c", res):
        assert p.read_bytes() == b""


@pytest.mark.parametrize("hw,net_hw", [((37, 53), (64, 96)), ((75, 124), (48, 160)), ((40, 40), (40, 40))])
def test_gray_restatement_equals_repmat(hw, net_hw):
    """imresize works per channel: resizing the one channel and writing it into the three BGR planes (each minus its
    own mean) is the repmat'ed frame's pre-processing, bit for bit."""
    from oracle import port
    rng = np.random.default_rng(hw[0])
    gray = rng.integers(0, 256, size=hw, dtype=np.uint8)
    want = port.preprocess(np.repeat(gray[:, :, None], 3, axis=2), net_hw)
    r = port.imresize(gray[:, :, None], net_hw)                  # [H][W][1]
    mean = np.asarray([104.0, 117.0, 123.0], dtype=np.float32)
    got = np.stack([r[:, :, 0].astype(np.float32) - mean[c] for c in range(3)])
    assert got.dtype == want.dtype and got.tobytes() == want.tobytes()


def test_channel_counts_other_than_1_and_3_are_refused_without_cuda():
    from mscnn_b200 import capi, ops
    L = capi.lib()
    INV = capi.ERR_INVALID
    plan = C.create_string_buffer(64)                   # never dereferenced on these paths
    fake = 0x1000
    hw = np.array([[375, 1242], [370, 1224]], np.int32)
    for bad in (2, 4, 0, -1):
        ch = np.array([3, bad], np.int32)
        for f in (L.mscnn_preprocess_forward_sized_c, L.mscnn_preprocess_forward_sized_c_host):
            assert f(plan, 2, hw.ctypes.data, ch.ctypes.data, fake, fake, None) == INV, bad
        from mscnn_b200 import net as mnet
        mnet._declare(L)
        assert L.mscnn_net_set_input_images_sized_c(plan, b"data", plan, 2, hw.ctypes.data, ch.ctypes.data,
                                                    fake) == INV
        assert L.mscnn_net_set_input_images_sized_async(plan, b"data", plan, 2, hw.ctypes.data, ch.ctypes.data,
                                                        fake) == INV
    for f in (L.mscnn_preprocess_forward_sized_c, L.mscnn_preprocess_forward_sized_c_host):
        ok = np.array([1, 3], np.int32)
        assert f(None, 2, hw.ctypes.data, ok.ctypes.data, fake, fake, None) == INV
        assert f(plan, 2, None, ok.ctypes.data, fake, fake, None) == INV
        assert f(plan, 2, hw.ctypes.data, ok.ctypes.data, None, fake, None) == INV
    for shape in ((5, 6, 2), (5, 6, 4)):
        with pytest.raises(AssertionError):
            ops.image_sizes_channels([np.zeros(shape, np.uint8)])
    hw2, ch2 = ops.image_sizes_channels([np.zeros((5, 6), np.uint8), np.zeros((7, 8, 1), np.uint8),
                                         np.zeros((9, 10, 3), np.uint8)])
    assert hw2.tolist() == [[5, 6], [7, 8], [9, 10]] and ch2.tolist() == [1, 1, 3]
