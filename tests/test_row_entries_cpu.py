"""Host-side argument checks of the row-count, multi-variant ROI pooling, head-tap and unfused-layer entries (no GPU):
every bad argument is refused with MSCNN_ERR_INVALID before any CUDA call, so the fake device pointers below are never
dereferenced."""
import ctypes as C

import pytest

FAKE = 0x1000          # a device pointer that is never touched on these paths
N, H, W, CH = 2, 6, 6, 64
R, P = 10, 7


def _lib():
    from mscnn_b200 import capi
    return capi, capi.lib()


def _roi_multi(L, nv, ratios, offs, x_lo=FAKE, y_lo=FAKE, ctot=2 * CH, dyn=False):
    r = (C.c_float * 8)(*ratios)
    o = (C.c_int * 8)(*offs)
    args = (FAKE, x_lo, N, H, W, CH, FAKE, R, P, P, 0.125, nv, C.cast(r, C.c_void_p), C.cast(o, C.c_void_p), FAKE, y_lo,
            ctot)
    if dyn:
        return L.mscnn_roi_pool_multi_forward_dyn(*args, FAKE, None)
    return L.mscnn_roi_pool_multi_forward(*args, None)


@pytest.mark.parametrize("dyn", [False, True], ids=["plain", "dyn"])
def test_roi_pool_multi_rejects_bad_arguments(dyn):
    capi, L = _lib()
    INV = capi.ERR_INVALID
    for nv in (0, 5):
        assert _roi_multi(L, nv, [0.0] * 8, [0] * 8, ctot=8 * CH, dyn=dyn) == INV, nv
    assert _roi_multi(L, 2, [0.0, 0.5], [0, CH + 4], dyn=dyn) == INV                 # offset not a multiple of 8
    assert _roi_multi(L, 2, [0.0, 0.5], [0, CH + 8], dyn=dyn) == INV                 # offset + C > out_channels
    assert _roi_multi(L, 1, [0.0], [CH + 8], ctot=2 * CH, dyn=dyn) == INV
    assert _roi_multi(L, 2, [0.0, 0.5], [0, CH], y_lo=None, dyn=dyn) == INV          # x_lo without y_lo
    assert _roi_multi(L, 2, [0.0, 0.5], [0, CH], x_lo=None, dyn=dyn) == INV          # y_lo without x_lo
    assert _roi_multi(L, 2, [0.0, 0.5], [0, CH], ctot=2 * CH + 4, dyn=dyn) == INV   # out_channels not a multiple of 8


def test_pool_dyn_rejects_bad_arguments():
    capi, L = _lib()
    INV = capi.ERR_INVALID
    f = L.mscnn_pool_forward_dyn
    assert f(FAKE, FAKE, FAKE, FAKE, N, H, W, CH, 2, 1, 2, FAKE, None) == INV        # pooling mode 2
    assert f(FAKE, FAKE, FAKE, FAKE, N, H, W, CH, 2, 1, -1, FAKE, None) == INV
    assert f(FAKE, FAKE, FAKE, None, N, H, W, CH, 2, 1, capi.POOL_MAX, FAKE, None) == INV   # x_lo without y_lo
    assert f(FAKE, None, FAKE, FAKE, N, H, W, CH, 2, 1, capi.POOL_MAX, FAKE, None) == INV
    assert f(FAKE, None, FAKE, None, N, H, W, CH + 4, 2, 1, capi.POOL_AVE, FAKE, None) == INV  # C % 8
    assert f(FAKE, None, FAKE, None, N, H, W, CH, 0, 1, capi.POOL_AVE, FAKE, None) == INV
    assert f(FAKE, None, FAKE, None, N, H, W, CH, 2, 0, capi.POOL_AVE, FAKE, None) == INV


def test_roi_align_dyn_rejects_bad_arguments():
    capi, L = _lib()
    INV = capi.ERR_INVALID

    def f(off, ctot, x_lo=FAKE, y_lo=FAKE):
        return L.mscnn_roi_align_forward_dyn(FAKE, x_lo, N, H, W, CH, FAKE, R, P, P, 0.125, 0.0, FAKE, y_lo, ctot, off,
                                             FAKE, None)
    assert f(4, 2 * CH) == INV                          # offset not a multiple of 8
    assert f(CH + 8, 2 * CH) == INV                     # offset + C > out_channels
    assert f(0, CH - 8) == INV
    assert f(CH, 2 * CH, y_lo=None) == INV              # x_lo without y_lo
    assert f(CH, 2 * CH, x_lo=None) == INV


def test_head_entries_reject_bad_arguments():
    capi, L = _lib()
    INV = capi.ERR_INVALID
    g = L.mscnn_head_gather
    assert g(FAKE, 64, FAKE, FAKE, N, H, W, 7, 5, 2, None) == INV       # only the 6- and 9-channel heads exist
    assert g(FAKE, 64, FAKE, FAKE, N, H, W, 0, 5, 2, None) == INV
    assert g(FAKE, 44, FAKE, FAKE, N, H, W, 9, 5, 2, None) == INV       # ld < k * Cout
    assert g(FAKE, 5 * 6 - 1, FAKE, FAKE, N, H, W, 6, 5, 2, None) == INV
    assert g(FAKE, 64, FAKE, FAKE, N, H, W, 9, 0, 0, None) == INV
    assert g(None, 64, FAKE, FAKE, N, H, W, 9, 5, 2, None) == INV
    p = L.mscnn_pack_head_weights
    assert p(FAKE, FAKE, FAKE, 9, CH, 7, 62, CH, None) == INV            # N_pad < k * Cout
    assert p(FAKE, FAKE, FAKE, 6, CH, 3, 17, CH, None) == INV
    assert p(FAKE, FAKE, FAKE, 9, CH, 5, 64, CH + 8, None) == INV       # Cin_pad % 64
    assert p(FAKE, FAKE, FAKE, 9, CH, 5, 64, CH - 64, None) == INV


def test_unfused_entries_reject_bad_arguments():
    capi, L = _lib()
    INV = capi.ERR_INVALID
    assert L.mscnn_relu_planes(FAKE, FAKE, 12, None) == INV                 # count % 8
    assert L.mscnn_relu_planes(None, FAKE, 16, None) == INV
    assert L.mscnn_relu_planes(FAKE, FAKE, 0, None) == capi.OK              # nothing to do, nothing launched
    assert L.mscnn_relu_f32(None, 16, None) == INV
    assert L.mscnn_relu_f32(FAKE, 0, None) == capi.OK
    cat = L.mscnn_concat_planes
    assert cat(FAKE, FAKE, 10, CH, 2 * CH, 4, None) == INV                  # offset not a multiple of 8
    assert cat(FAKE, FAKE, 10, CH, 2 * CH, CH + 8, None) == INV             # offset + C > Ctot
    assert cat(FAKE, FAKE, 10, CH + 4, 2 * CH, 0, None) == INV
    assert cat(FAKE, FAKE, 10, CH, 2 * CH + 4, 0, None) == INV
    assert cat(None, FAKE, 10, CH, 2 * CH, 0, None) == INV
    assert cat(FAKE, FAKE, 0, CH, 2 * CH, CH, None) == capi.OK
