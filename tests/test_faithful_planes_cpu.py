"""What tests/test_faithful_planes_gpu.py relies on, checked without a GPU: the inputs keep a live lo plane, hold ties in
hi inside pooling and ROI windows and halfway values; the store rounding is exact; the ROI set reaches odd, even and
empty bin windows; the fp32 depthwise restatement is the oracle's deconvolution bit for bit; and the restated global AVE
order stays within the bound DESIGN §4.1 states."""
import numpy as np
import pytest

import faithful_planes_ref as F
from deconv_ref import depthwise_col2im_f32
from oracle import port

SHAPES = [(2, 64, 24, 80), (2, 512, 9, 15), (1, 264, 7, 11)]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


@pytest.mark.parametrize("kind", ["signed", "relu"])
@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_inputs_keep_a_live_lo_plane(kind, shape):
    x = F.faithful_input(np.random.default_rng(1), shape, kind)
    hi, lo = F.split_planes(x)
    rep = hi + lo                                      # the value the planes hold: exact in fp32
    assert np.array_equal(rep.astype(np.float64), hi.astype(np.float64) + lo.astype(np.float64))
    assert float((lo != 0).mean()) >= 0.9
    assert bool(((hi * lo) < 0).any()) and bool(((hi * lo) > 0).any())   # lo of both signs
    if kind == "relu":
        assert 0.02 <= float((x == 0).mean()) <= 0.1 and float(x.min()) >= 0.0


@pytest.mark.parametrize("kind", ["signed", "relu"])
def test_inputs_hold_hi_ties_in_windows(kind):
    """2x2 / 2 windows whose two largest values share hi and differ in lo: many, in every channel (so in both channel
    groups of a lane at C = 512), and with lo of either sign at the maximum."""
    x = F.faithful_input(np.random.default_rng(2), (2, 512, 24, 80), kind)
    hi, lo = F.split_planes(x)
    n, c, h, w = x.shape
    win = lambda a: a.reshape(n, c, h // 2, 2, w // 2, 2).transpose(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
    v, vh, vl = win(x), win(hi), win(lo)
    order = np.argsort(-v, axis=-1)
    top = np.take_along_axis(vh, order[..., :2], -1)
    tied = (top[..., 0] == top[..., 1]) & (np.take_along_axis(vl, order[..., :1], -1)[..., 0] !=
                                           np.take_along_axis(vl, order[..., 1:2], -1)[..., 0])
    assert int(tied.sum()) >= 2 * 6 * 4 * c               # six 4x4 patches per image: four tied windows each
    for ch in (0, 255, 256, 511):
        assert bool(tied[:, ch].any()), ch
    best_lo = np.take_along_axis(vl, order[..., :1], -1)[..., 0][tied]
    assert bool((best_lo > 0).any()) and bool((best_lo < 0).any())


def test_inputs_hold_halfway_values():
    x = F.faithful_input(np.random.default_rng(3), (2, 64, 24, 80), "signed")
    hi, lo = F.split_planes(x)
    nz = hi != 0
    half = nz & (np.abs(lo) == F.half_ulp(np.where(nz, hi, 1)))
    assert float(half.mean()) >= 0.02
    assert bool((lo[half] > 0).any()) and bool((lo[half] < 0).any())
    assert bool((np.signbit(x) & (x == 0)).any())        # -0.0 inputs


def test_store_rounding_is_exact():
    rng = np.random.default_rng(4)
    r = np.concatenate([rng.standard_normal(20000).astype(np.float32) * np.float32(2.0 ** rng.integers(-20, 20)),
                        F.faithful_input(rng, (1, 8, 8, 8), "signed").reshape(-1),
                        np.array([0.0, -0.0, 1.0, 3.0e38, -1e-30], np.float32)])
    s = F.stored(r, True)
    hi, lo = F.split_planes(r)
    # hi' + lo' is an fp32 value (the fp32 sum is exact), and storing it again keeps it
    assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), s.astype(np.float64))
    assert np.array_equal(F.stored(s, True), s)
    # hi' + lo' keeps 16 significant bits: within 2^-16 relative of r
    nz = r != 0
    assert bool((np.abs(s[nz].astype(np.float64) - r[nz]) <= 2.0 ** -16 * np.abs(r[nz])).all())
    b = F.stored(r, False)
    assert np.array_equal(_bits(b), _bits(hi)) and np.array_equal(_bits(F.stored(b, False)), _bits(b))


def test_roi_set_reaches_odd_even_and_empty_windows():
    rng = np.random.default_rng(5)
    h, w = 24, 40
    for scale in (0.125, 0.25):
        rois = F.special_rois(rng, 2, w / scale, h / scale, 120)
        for bins in [(7, 7), (5, 5), (8, 4), (1, 7)]:
            for pr in (0.0, 0.25):
                npx = F.roi_pool_windows(rois, h, w, *bins, scale, pr)
                assert (npx == 0).any() and (npx == 1).any(), (scale, bins, pr)
                assert ((npx >= 3) & (npx % 2 == 1)).any() and ((npx >= 2) & (npx % 2 == 0)).any(), (scale, bins, pr)
                assert (npx[2] == 0).all()                    # the ROI outside the image: every bin empty


def test_roi_windows_match_the_oracle():
    """The restated bin windows are empty exactly where the oracle's are: pooling a map of ones gives 1 in a non-empty
    bin and 0 in an empty one.  (Guards the geometry the coverage check above relies on.)"""
    rng = np.random.default_rng(6)
    h, w = 12, 20
    rois = F.special_rois(rng, 1, w / 0.125, h / 0.125, 60)
    npx = F.roi_pool_windows(rois, h, w, 7, 7, 0.125, 0.25)
    ones = port.roi_pool(np.ones((1, 1, h, w), np.float32), rois, 7, 7, 0.125, 0.25)[:, 0]
    assert np.array_equal(ones == 1, npx > 0)


DW_GEOMS = [(4, 2, 1), (8, 4, 2), (16, 8, 4), (2, 2, 0), (3, 1, 1), (5, 3, 1), (1, 8, 0), (12, 6, 3)]


@pytest.mark.parametrize("k,stride,pad", DW_GEOMS, ids=[f"k{k}s{s}p{p}" for k, s, p in DW_GEOMS])
def test_depthwise_restatement_is_the_oracle(k, stride, pad):
    rng = np.random.default_rng(7 + k)
    x = F.faithful_input(rng, (2, 16, 7, 9), "signed")
    wt = rng.standard_normal((16, 1, k, k)).astype(np.float32)
    got = depthwise_col2im_f32(x, wt, None, stride, pad)
    ref = port.deconv_depthwise(x, wt, stride, pad)
    assert np.array_equal(_bits(got), _bits(ref))


def test_depthwise_restatement_with_bias_and_dilation_against_fp64():
    """Where the oracle has no geometry (rectangular, dilated, bias): within the fp32 rounding of a short sum."""
    from deconv_ref import scatter_deconv
    rng = np.random.default_rng(8)
    x = rng.standard_normal((2, 8, 6, 7)).astype(np.float32)
    wt = rng.standard_normal((8, 1, 3, 6)).astype(np.float32)
    b = rng.standard_normal(8).astype(np.float32)
    got = depthwise_col2im_f32(x, wt, b, (2, 4), (1, 2), (2, 1))
    ref = scatter_deconv(x, wt, (2, 4), (1, 2), (2, 1), group=8, bias=b)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 2.0 ** -20 * (np.abs(ref).max() + 1)


@pytest.mark.parametrize("hw", [(4, 8), (9, 11), (24, 80), (50, 80)])
def test_global_ave_order_within_the_stated_bound(hw):
    """The kernel's slice order lands within (HW - 1) 2^-24 mean|x| (+ the division's rounding) of the exact mean."""
    rng = np.random.default_rng(9)
    x = F.faithful_input(rng, (2, 64, *hw), "relu")
    got = F.global_ave_kernel_order(x).astype(np.float64)
    exact = x.astype(np.float64).mean(axis=(2, 3), keepdims=True)
    n = hw[0] * hw[1]
    bound = (n - 1) * 2.0 ** -24 * np.abs(x).astype(np.float64).mean(axis=(2, 3), keepdims=True) + 2.0 ** -24 * np.abs(exact)
    assert bool((np.abs(got - exact) <= bound).all())
