"""Host-side checks of Deconvolution with any kernel, stride, pad, dilation, group and bias: the phase decomposition
mscnn_deconv_forward runs (restated in numpy against the direct scatter), the phase plans it reports
(mscnn_deconv_plan_describe, no device), the packed-weight size, the shapes a Net derives, the CHECKs for what is not
served, and torch's fp64 conv_transpose2d against the reference's own Deconvolution layer where oracle/_ref is built."""
import ctypes as C
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from deconv_ref import DECONV_SIZES, axis_phase, deconv_net, deconv_out, packed_elems, phase_deconv, scatter_deconv

ROOT = Path(__file__).resolve().parents[1]
FAKE = 0x10000   # never dereferenced: the plan query makes no CUDA call


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


# ---- the phase decomposition, restated ----
GRID = [(k, s, p, d) for k in (1, 2, 3, 4, 5, 8) for s in (1, 2, 3, 4, 8) for p in (0, 1, 2, 3, 5) for d in (1, 2, 3)]


def test_phase_decomposition_equals_the_scatter_deconvolution():
    """Over kernels, strides, pads and dilations that include k < s, gcd(s, d) > 1 (phases no tap reaches),
    p > d (k - 1) (a negative sub-pad) and odd output extents: every phase's stride-1 convolution gives the scatter."""
    rng = np.random.default_rng(1)
    seen = dict(k_below_s=0, tapless=0, negative_pad=0, odd=0)
    for k, s, p, d in GRID:
        for h, w in [(5, 4), (3, 7)]:
            ho, wo = deconv_out(h, k, s, p, d), deconv_out(w, k, s, p, d)
            if ho <= 0 or wo <= 0:
                continue
            x = rng.standard_normal((2, 3, h, w))
            wt = rng.standard_normal((3, 2, k, k))
            b = rng.standard_normal(2)
            want = scatter_deconv(x, wt, s, p, d, 1, b)
            got = phase_deconv(x, wt, s, p, d, 1, b)
            assert got.shape == want.shape == (2, 2, ho, wo)
            assert np.allclose(got, want, rtol=1e-12, atol=1e-12), (k, s, p, d, h, w)
            phases = [axis_phase(k, s, p, d, ho, r) for r in range(s)]
            seen["k_below_s"] += k < s
            seen["tapless"] += any(not t for t, _, _, q in phases if q)
            seen["negative_pad"] += any(pad < 0 for t, _, pad, _ in phases if t)
            seen["odd"] += ho % 2
    assert all(v > 0 for v in seen.values()), seen


def test_phase_decomposition_rectangular_and_grouped():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((2, 8, 5, 6))
    for group in (1, 2, 4):
        for k, s, p, d in [((3, 2), (2, 3), (1, 0), (1, 2)), ((4, 1), (3, 1), (2, 0), (2, 1)), ((2, 5), (1, 4), (0, 3), 1)]:
            wt = rng.standard_normal((8, 12 // group) + _pair(k))
            assert np.allclose(phase_deconv(x, wt, s, p, d, group), scatter_deconv(x, wt, s, p, d, group),
                               rtol=1e-12, atol=1e-12), (group, k, s, p, d)


def test_every_tap_lies_in_exactly_one_phase():
    for k, s, p, d in GRID:
        taps = sorted(t for r in range(s) for t in axis_phase(k, s, p, d, 0, r)[0])
        assert taps == list(range(k)), (k, s, p, d)


# ---- plans and packing (host-only C entries) ----
def _desc(n, cin, h, w, cout, k, stride, pad, dil=1, group=1, split=True):
    from mscnn_b200 import capi
    d = capi.ConvDesc()
    d.x_hi, d.x_lo = FAKE, (FAKE if split else None)
    d.N, d.H, d.W, d.C = n, h, w, (cin + 63) // 64 * 64
    d.w_hi, d.w_lo, d.bias = FAKE, (FAKE if split else None), FAKE
    d.Cout, d.Cout_pad = cout, (cout + 63) // 64 * 64
    (d.KH, d.KW), (d.pad_h, d.pad_w) = _pair(k), _pair(pad)
    (d.stride_h, d.stride_w), (d.dil_h, d.dil_w), d.group = _pair(stride), _pair(dil), group
    d.out_mode = capi.OUT_NHWC_BF16
    d.y_hi, d.y_lo = FAKE, (FAKE if split else None)
    return d


def _describe(d):
    from mscnn_b200 import capi
    buf = C.create_string_buffer(1 << 14)
    rc = capi.lib().mscnn_deconv_plan_describe(C.byref(d), buf, 1 << 14)
    return rc, buf.value.decode()


def _phases(text):
    out = []
    for line in text.strip().split("\n"):
        head, plan = line.split(" plan=", 1)
        f = dict(kv.split("=") for kv in head.split(" "))
        out.append((f, plan))
    return out


DESCRIBE_CASES = [
    # N, Cin, H, W, Cout, k, stride, pad, dil, group
    (8, 512, 48, 160, 512, 4, 2, 1, 1, 1),
    (8, 256, 96, 320, 256, 2, 2, 0, 1, 1),
    (1, 64, 5, 7, 24, 1, 4, 0, 1, 1),
    (1, 64, 5, 7, 64, 3, 2, 2, 2, 1),
    (2, 128, 9, 30, 128, (3, 5), (2, 3), (4, 0), (1, 2), 2),
    (1, 64, 6, 64, 64, 3, 1, 1, 1, 1),
    (3, 64, 4, 5, 128, 8, 8, 3, 3, 1),
]


@pytest.mark.parametrize("case", DESCRIBE_CASES, ids=lambda c: "x".join(map(str, c[5:9])))
def test_plan_lists_the_phases_the_restatement_predicts(case):
    n, cin, h, w, cout, k, s, p, d, g = case
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = _pair(k), _pair(s), _pair(p), _pair(d)
    rc, text = _describe(_desc(n, cin, h, w, cout, k, s, p, d, g))
    assert rc == 0, text
    lines = _phases(text)
    ho, wo = deconv_out(h, kh, sh, ph, dh), deconv_out(w, kw, sw, pw, dw)
    assert len(lines) == sh * sw
    for i, (f, plan) in enumerate(lines):
        th, dil_h, pad_h, qh = axis_phase(kh, sh, ph, dh, ho, i // sw)
        tw, dil_w, pad_w, qw = axis_phase(kw, sw, pw, dw, wo, i % sw)
        assert f["phase"] == f"{i // sw}x{i % sw}"
        assert f["taps"] == f"{len(th)}x{len(tw)}" and f["out"] == f"{qh}x{qw}"
        if th and tw:
            assert f["dil"] == f"{dil_h}x{dil_w}" and f["pad"] == f"{pad_h}x{pad_w}"
        if qh == 0 or qw == 0:
            assert plan == "none"
        elif not th or not tw:
            assert plan == "bias_fill"
        else:
            assert plan.startswith("kernel=conv_igemm_kernel<") and "stride=" not in plan.replace("stride=1x1", "")


def test_pinned_plan_strings():
    # the dense 4 / 2 / 1 layer on conv5_3 of a full-size batch (512 -> 512, 48 x 160): four phases of 2 x 2 taps, one per
    # parity of the output, pads 1 / 0 by parity
    _, text = _describe(_desc(8, 512, 48, 160, 512, 4, 2, 1))
    lines = _phases(text)
    plan = ("kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 "
            "rowshare=0 a_stages=0")
    assert [(f["phase"], f["taps"], f["pad"], f["out"], p) for f, p in lines] == [
        ("0x0", "2x2", "1x1", "48x160", plan), ("0x1", "2x2", "1x0", "48x160", plan),
        ("1x0", "2x2", "0x1", "48x160", plan), ("1x1", "2x2", "0x0", "48x160", plan)]
    # the shipped -2x layer's shape as a dense layer (conv4_3, 512 -> 512 at 96 x 320, batch 1)
    _, text = _describe(_desc(1, 512, 96, 320, 512, 4, 2, 1))
    assert _phases(text)[0][1] == ("kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 "
                                   "epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0")
    # a stride-1 3 x 3 deconvolution on 64-pixel rows takes the shared haloed row
    _, text = _describe(_desc(1, 64, 6, 64, 64, 3, 1, 1))
    assert _phases(text)[0][1].endswith("rowshare=1 a_stages=2") and _phases(text)[0][0]["pad"] == "1x1"
    # dilation 2 at stride 2: only the even phase has taps, the rest hold the bias
    _, text = _describe(_desc(1, 64, 5, 7, 64, 3, 2, 2, 2))
    assert [p for _, p in _phases(text)][1:] == ["bias_fill"] * 3


def test_rowshare_with_a_negative_sub_pad():
    """k6 / s2 / p6: each phase is a 3-tap stride-1 convolution with pad -1 in both axes; on 128-pixel rows it takes the
    row-share plan (one haloed activation row from column w0 + 1)."""
    _, text = _describe(_desc(1, 64, 8, 132, 64, 6, 2, 6))
    for f, plan in _phases(text):
        assert f["taps"] == "3x3" and f["pad"] == "-1x-1" and f["out"] == "4x128", f
        assert "rowshare=1" in plan, plan


UNSERVED = [
    ("stride9", dict(stride=9)),
    ("group_32", dict(cin=64, cout=64, group=2)),
    ("group_not_dividing", dict(cin=128, cout=192, group=2)),
    ("extent_not_positive", dict(h=1, w=1, k=1, pad=1)),
    ("negative_pad", dict(pad=-1)),
    ("zero_kernel", dict(k=0)),
]


@pytest.mark.parametrize("case", UNSERVED, ids=[c[0] for c in UNSERVED])
def test_unserved_geometries_are_refused_with_a_message(case):
    from mscnn_b200 import capi
    args = dict(n=1, cin=128, h=8, w=8, cout=128, k=3, stride=2, pad=1, dil=1, group=1)
    args.update(case[1])
    code = ("import ctypes as C, sys\nsys.path.insert(0, 'tests')\nfrom test_deconv_cpu import _desc, _describe\n"
            f"print(_describe(_desc(**{args!r}))[0])")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=str(ROOT))
    assert r.stdout.strip() == str(capi.ERR_INVALID), r.stdout + r.stderr
    if case[0] not in ("negative_pad", "zero_kernel", "extent_not_positive"):
        assert "mscnn_deconv_forward:" in r.stderr, r.stderr
    assert _describe(_desc(**args))[0] == capi.ERR_INVALID


def test_other_outputs_are_refused():
    from mscnn_b200 import capi
    for field, value in [("out_mode", capi.OUT_NCHW_F32), ("pool_hi", FAKE), ("dyn_n", FAKE)]:
        d = _desc(1, 64, 8, 8, 64, 4, 2, 1)
        setattr(d, field, value)
        assert _describe(d)[0] == capi.ERR_INVALID, field


@pytest.mark.parametrize("geom", [(512, 512, 1, 4, 2, 1, 1), (256, 256, 1, 2, 2, 0, 1), (64, 24, 1, 1, 4, 0, 1),
                                  (128, 256, 2, (3, 5), (2, 3), (4, 0), (1, 2)), (64, 64, 1, 3, 2, 2, 2),
                                  (100, 70, 1, 8, 8, 3, 3), (256, 128, 4, 5, 3, 1, 2)])
def test_packed_elems_match_the_restatement(geom):
    from mscnn_b200 import capi
    cin, cout, g, k, s, p, d = geom
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = _pair(k), _pair(s), _pair(p), _pair(d)
    got = capi.lib().mscnn_deconv_packed_elems(cin, cout, g, kh, kw, sh, sw, ph, pw, dh, dw, (cout + 63) // 64 * 64)
    assert got == packed_elems(cin, cout, g, k, s, p, d) == kh * kw * ((cout + 63) // 64 * 64) * ((cin // g + 63) // 64 * 64)
    assert capi.lib().mscnn_deconv_packed_elems(cin, cout, g, kh, kw, 9, sw, ph, pw, dh, dw, 64 * cout) == -1


# ---- shapes through a Net (no forward) ----
def _net_text(body, c=64, h=20, w=30):
    return f'input: "d" input_dim: 2 input_dim: {c} input_dim: {h} input_dim: {w}\n' + body


def _deconv_layer(param, cout=64):
    return (f'layer {{ name: "u" type: "Deconvolution" bottom: "d" top: "u" '
            f'convolution_param {{ num_output: {cout} {param} }} }}\n')


NET_SHAPES = [
    # prototxt fields, Cin, Cout, group, (kh, kw), (sh, sw), (ph, pw), (dh, dw), bias
    ("kernel_size: 4 stride: 2 pad: 1 group: 64 bias_term: false", 64, 64, 64, (4, 4), (2, 2), (1, 1), (1, 1), False),
    ("kernel_size: 4 stride: 2 pad: 1", 64, 512, 1, (4, 4), (2, 2), (1, 1), (1, 1), True),
    ("kernel_h: 3 kernel_w: 5 stride_h: 2 stride_w: 3 pad_h: 1 pad_w: 0", 64, 64, 1, (3, 5), (2, 3), (1, 0), (1, 1), True),
    ("kernel_size: 3 stride: 2 pad: 2 dilation: 2 bias_term: true", 64, 32, 1, (3, 3), (2, 2), (2, 2), (2, 2), True),
    ("kernel_size: 3 stride: 1 pad: 0 dilation: 3 dilation: 1", 64, 64, 1, (3, 3), (1, 1), (0, 0), (3, 1), True),
    ("kernel_size: 2 stride: 2 group: 2", 128, 256, 2, (2, 2), (2, 2), (0, 0), (1, 1), True),
    ("kernel_size: 16 stride: 8 pad: 4 group: 64 bias_term: false", 64, 64, 64, (16, 16), (8, 8), (4, 4), (1, 1), False),
    ("kernel_size: 3 stride: 8 pad: 0", 64, 24, 1, (3, 3), (8, 8), (0, 0), (1, 1), True),
]


@pytest.mark.parametrize("hw", [(20, 30), (7, 9)], ids=["even", "odd"])
@pytest.mark.parametrize("case", NET_SHAPES, ids=[re.sub(r"[: ]+", "_", c[0]) for c in NET_SHAPES])
def test_deconvolution_top_and_blob_shapes(case, hw):
    from mscnn_b200.net import Net
    param, cin, cout, g, k, s, p, d, bias = case
    h, w = hw
    net = Net(_net_text(_deconv_layer(param, cout), c=cin, h=h, w=w))
    assert net.blob_shape("u") == (2, cout, deconv_out(h, k[0], s[0], p[0], d[0]), deconv_out(w, k[1], s[1], p[1], d[1]))
    assert net.param_shapes("u") == [(cin, cout // g) + k] + ([(cout,)] if bias else [])


def test_deconv_net_shapes():
    from mscnn_b200.net import Net
    for h, w in DECONV_SIZES:
        net = Net(deconv_net(h, w))
        h1, w1 = (h + 1) // 2, (w + 1) // 2
        assert net.blob_shape("d_dense") == (2, 128, 2 * h1, 2 * w1) == net.blob_shape("d_group")[:1] + (128, 2 * h1, 2 * w1)
        assert net.blob_shape("cat_up") == (2, 256, 2 * h1, 2 * w1)
        assert net.blob_shape("d_dw") == (2, 16, 8 * h1, 8 * w1) and net.blob_shape("c4") == (2, 64, 2 * h1, 2 * w1)
        assert net.blob_shape("d_odd") == net.blob_shape("d_dil") == (2, 32, 4 * h1 - 1, 4 * w1 - 1)
        assert net.blob_shape("cat_odd") == (2, 64, 4 * h1 - 1, 4 * w1 - 1)
        assert net.param_shapes("d_dense") == [(128, 128, 4, 4), (128,)] and net.param_shapes("d_group") == [(128, 64, 2, 2)]
        assert net.param_shapes("d_dw") == [(16, 1, 8, 8)] and net.param_shapes("d_dil") == [(64, 32, 3, 3), (32,)]


ABORTS = [
    ("stride_9", _net_text(_deconv_layer("kernel_size: 4 stride: 9")), "strides 1..8"),
    ("group_32_channels", _net_text(_deconv_layer("kernel_size: 4 stride: 2 group: 2")), "multiples of 64"),
    ("channel_multiplier", _net_text(_deconv_layer("kernel_size: 4 stride: 2 group: 64", cout=128)), "channel multiplier"),
    ("group_not_dividing", _net_text(_deconv_layer("kernel_size: 4 group: 5", cout=65)), "channels_ % group_"),
    ("extent_not_positive", _net_text(_deconv_layer("kernel_size: 1 pad: 1"), h=1, w=1), "is not positive"),
    ("kernel_twice", _net_text(_deconv_layer("kernel_size: 3 kernel_h: 3 kernel_w: 3")), "Either kernel_size or kernel_h/w"),
    ("dilation_three_times", _net_text(_deconv_layer("kernel_size: 3 dilation: 1 dilation: 1 dilation: 1")), "dilation must be"),
]


@pytest.mark.parametrize("case", ABORTS, ids=[c[0] for c in ABORTS])
def test_rejected_geometries_abort_with_their_message(case):
    _, text, message = case
    r = subprocess.run([sys.executable, "-c", "import sys; from mscnn_b200.net import Net; Net(sys.argv[1])", text],
                       capture_output=True, text=True, cwd=str(ROOT))
    assert r.returncode != 0 and message in r.stderr, r.stderr[-600:]


# ---- torch's fp64 conv_transpose2d against the reference's own layer ----
@pytest.fixture(scope="module")
def ref_built():
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref is not built (needs the reference sources)")


REF_CASES = [
    # prototxt fields, Cin, Cout, group, kernel, stride, pad, dilation, bias
    ("kernel_size: 4 stride: 2 pad: 1", 8, 6, 1, (4, 4), (2, 2), (1, 1), (1, 1), True),
    ("kernel_size: 2 stride: 2 group: 2 bias_term: false", 8, 6, 2, (2, 2), (2, 2), (0, 0), (1, 1), False),
    ("kernel_size: 8 stride: 4 pad: 2 group: 8 bias_term: false", 8, 8, 8, (8, 8), (4, 4), (2, 2), (1, 1), False),
    ("kernel_size: 3 stride: 2 pad: 1", 8, 6, 1, (3, 3), (2, 2), (1, 1), (1, 1), True),
    ("kernel_size: 3 stride: 2 pad: 2 dilation: 2", 8, 6, 1, (3, 3), (2, 2), (2, 2), (2, 2), True),
    ("kernel_h: 3 kernel_w: 5 stride_h: 2 stride_w: 3 pad_h: 1 pad_w: 0", 8, 6, 1, (3, 5), (2, 3), (1, 0), (1, 1), True),
    ("kernel_size: 2 stride: 4 pad: 0", 8, 6, 1, (2, 2), (4, 4), (0, 0), (1, 1), True),
    ("kernel_size: 3 stride: 1 pad: 4 dilation: 3 dilation: 1 group: 2", 8, 6, 2, (3, 3), (1, 1), (4, 4), (3, 1), True),
]


@pytest.mark.parametrize("case", REF_CASES, ids=[re.sub(r"[: ]+", "_", c[0]) for c in REF_CASES])
def test_torch_fp64_deconvolution_matches_the_reference_layer(ref_built, case):
    """The GPU tests compare with torch's fp64 conv_transpose2d; here that reference and the numpy scatter are held to
    DeconvolutionLayer::Forward_cpu (fp32 gemm + col2im): 1e-4 of the output's rms."""
    import torch
    import torch.nn.functional as F
    from oracle import ref
    param, cin, cout, g, k, s, p, d, bias = case
    rng = np.random.default_rng(21)
    x = rng.standard_normal((2, cin, 9, 11)).astype(np.float32)
    w = (rng.standard_normal((cin, cout // g) + k) * 0.2).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    net = ref.RefNet(_net_text(_deconv_layer(param, cout), c=cin, h=9, w=11))
    net.set_params({"u": [w, b] if bias else [w]})
    net.set_blob("d", x)
    net.forward()
    got = net.blob("u")
    want = F.conv_transpose2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(),
                              torch.from_numpy(b).double() if bias else None, stride=s, padding=p, dilation=d,
                              groups=g).numpy()
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-4 * np.sqrt((want ** 2).mean())
    assert np.allclose(scatter_deconv(x, w, s, p, d, g, b if bias else None), want, rtol=1e-10, atol=1e-10)
