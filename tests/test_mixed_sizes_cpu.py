"""Batches of images with different original sizes, host side (no GPU): the per-image geometry helper
(mscnn_detect_image_geometry) gives exactly the fp32 ratios and sizes that kitti_detect_cfg stores for one image
(examples/kitti_car/run_mscnn_detection.m:64-65), and every new entry rejects bad arguments before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

KITTI_SIZES = [(375, 1242), (370, 1224), (374, 1238), (376, 1241), (1, 1), (7, 3000)]


@pytest.mark.parametrize("net_hw", [(768, 2560), (576, 1920), (384, 1280)])
def test_image_geometry_equals_kitti_detect_cfg(net_hw):
    from mscnn_b200 import net as mnet
    sizes = KITTI_SIZES + [net_hw]                      # org == net: both ratios exactly 1
    g = mnet.image_geometry(net_hw, sizes)
    assert g.dtype == np.float32 and g.shape == (len(sizes), 4)
    for n, org in enumerate(sizes):
        cfg = mnet.kitti_detect_cfg(*net_hw, org_hw=org)
        want = np.array([cfg.ratio_h, cfg.ratio_w, cfg.org_h, cfg.org_w], dtype=np.float32)
        assert g[n].tobytes() == want.tobytes(), (net_hw, org, g[n], want)
    assert np.all(g[-1, :2] == 1.0)


def test_new_entries_reject_bad_arguments_without_cuda():
    from mscnn_b200 import capi
    L = capi.lib()
    INV = capi.ERR_INVALID
    out = np.zeros((2, 4), np.float32)
    good = np.array([[375, 1242], [370, 1224]], np.int32)
    bad = np.array([[375, 1242], [0, 1224]], np.int32)
    assert L.mscnn_detect_image_geometry(768, 2560, 2, good.ctypes.data, out.ctypes.data) == capi.OK
    assert L.mscnn_detect_image_geometry(768, 2560, 2, bad.ctypes.data, out.ctypes.data) == INV
    assert L.mscnn_detect_image_geometry(0, 2560, 2, good.ctypes.data, out.ctypes.data) == INV
    assert L.mscnn_detect_image_geometry(768, 2560, 0, good.ctypes.data, out.ctypes.data) == INV
    assert L.mscnn_detect_image_geometry(768, 2560, 2, None, out.ctypes.data) == INV
    assert L.mscnn_detect_image_geometry(768, 2560, 2, good.ctypes.data, None) == INV

    # pre-processing: arguments are checked before the plan or the device is touched
    plan = C.create_string_buffer(64)                   # never dereferenced on these paths
    fake = 0x1000
    for f in (L.mscnn_preprocess_forward_sized, L.mscnn_preprocess_forward_sized_host):
        assert f(None, 2, good.ctypes.data, fake, fake, None) == INV
        assert f(plan, 0, good.ctypes.data, fake, fake, None) == INV
        assert f(plan, 2, None, fake, fake, None) == INV
        assert f(plan, 2, bad.ctypes.data, fake, fake, None) == INV
        assert f(plan, 2, good.ctypes.data, None, fake, None) == INV
        assert f(plan, 2, good.ctypes.data, fake, None, None) == INV

    # post-process: a missing, zero, negative, NaN or infinite geometry value is refused
    from mscnn_b200 import net as mnet
    cfg = mnet.kitti_detect_cfg(768, 2560)
    geo = mnet.image_geometry((768, 2560), good)
    dev = [fake] * 5
    for name in ("mscnn_detect_postprocess_sized", "mscnn_cascade_detect_postprocess_sized"):
        f = getattr(L, name)
        assert f(cfg, 2, *dev, 1 << 20, fake, fake, None, None) == INV
        for v in (0.0, -1.0, np.nan, np.inf):
            g = geo.copy()
            g[1, 2] = v
            assert f(cfg, 2, *dev, 1 << 20, fake, fake, g.ctypes.data, None) == INV, (name, v)
    assert L.mscnn_detect_postprocess_packed_sized(cfg, 2, *dev, 1 << 20, fake, None, None) == INV
    assert L.mscnn_detect_postprocess_packed_sized(cfg, 2, *dev, 1 << 20, None, geo.ctypes.data, None) == INV
