"""Host-side checks of the convolution geometries beyond stride 1 / dilation 1 / group 1 and of the pooling geometries
beyond square / pad 0: the launch plan (mscnn_conv_plan_describe, no device), the layer shapes a Net derives, the CHECKs
that remain, and the test references against the reference's own layers where oracle/_ref is built."""
import ctypes as C
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from conv_geometry_ref import GEOMETRY_SIZES, conv_out, geometry_net, pool, pooled

ROOT = Path(__file__).resolve().parents[1]
FAKE = 0x10000   # never dereferenced: the plan query makes no CUDA call


def _desc(n, cin, h, w, cout, kh, kw, pad, split=True, pooled_out=False, **geom):
    from mscnn_b200 import capi
    d = capi.ConvDesc()
    d.x_hi, d.x_lo = FAKE, (FAKE if split else None)
    d.N, d.H, d.W, d.C = n, h, w, (cin + 63) // 64 * 64
    d.w_hi, d.w_lo, d.bias = FAKE, (FAKE if split else None), FAKE
    d.Cout, d.Cout_pad, d.KH, d.KW = cout, (cout + 63) // 64 * 64, kh, kw
    d.pad_h, d.pad_w = pad if isinstance(pad, tuple) else (pad, pad)
    d.out_mode = capi.OUT_NHWC_BF16
    if pooled_out:
        d.pool_hi, d.pool_lo = FAKE, (FAKE if split else None)
    else:
        d.y_hi, d.y_lo = FAKE, (FAKE if split else None)
    for k, v in geom.items():
        setattr(d, k, v)
    return d


def _describe(d):
    from mscnn_b200 import capi
    buf = C.create_string_buffer(512)
    rc = capi.lib().mscnn_conv_plan_describe(C.byref(d), buf, 512)
    return rc, buf.value.decode()


def _fields(text):
    return dict(kv.split("=", 1) for kv in re.split(r" (?=[a-z_]+=)", text))


def test_unset_and_unit_geometry_give_todays_plan_string():
    for args in [(8, 512, 96, 320, 512, 3, 3, 1), (2, 64, 384, 1280, 128, 3, 3, 1), (4, 128, 7, 7, 128, 3, 3, 0)]:
        rc0, plain = _describe(_desc(*args))
        rc1, ones = _describe(_desc(*args, stride_h=1, stride_w=1, dil_h=1, dil_w=1, group=1))
        assert rc0 == 0 and rc1 == 0 and plain == ones
        assert "stride=" not in plain and "group=" not in plain and plain.endswith(f"a_stages={_fields(plain)['a_stages']}")


PLAN_CASES = [
    # name, args, geometry, kernel instantiation
    ("s2_512", (8, 512, 96, 320, 512, 3, 3, 1), dict(stride_h=2, stride_w=2), "conv_igemm_kernel<256, false>"),
    ("s4_wide", (1, 64, 64, 2048, 64, 3, 3, 1), dict(stride_h=4, stride_w=4), "conv_igemm_kernel<64, true>"),
    ("s3_wide", (1, 64, 9, 1500, 128, 3, 3, 1), dict(stride_h=3, stride_w=3), "conv_igemm_kernel<128, true>"),
    ("s1x2", (2, 64, 8, 1024, 64, 3, 3, 1), dict(stride_h=1, stride_w=2), "conv_igemm_kernel<64, true>"),
    ("s2x1", (2, 64, 8, 256, 64, 3, 3, 1), dict(stride_h=2, stride_w=1), "conv_igemm_kernel<64, true>"),
    ("dil2", (8, 512, 48, 160, 512, 3, 3, 2), dict(dil_h=2, dil_w=2), "conv_igemm_kernel<256, false>"),
    ("dil2_w128", (1, 64, 6, 256, 64, 3, 3, 2), dict(dil_h=2, dil_w=2), "conv_igemm_kernel<64, true>"),
    ("dil2x1_w128", (1, 64, 6, 256, 64, 3, 3, (2, 1)), dict(dil_h=2, dil_w=1), "conv_igemm_kernel<64, true>"),
    ("g4_512", (8, 512, 96, 320, 512, 3, 3, 1), dict(group=4), "conv_igemm_kernel<128, true>"),
    ("g8_512", (8, 512, 96, 320, 512, 3, 3, 1), dict(group=8), "conv_igemm_kernel<64, true>"),
    ("g2_512", (8, 512, 96, 320, 512, 3, 3, 1), dict(group=2), "conv_igemm_kernel<256, false>"),
    ("g2_128_256", (1, 128, 12, 40, 256, 3, 3, 1), dict(group=2), "conv_igemm_kernel<128, true>"),
]


@pytest.mark.parametrize("case", PLAN_CASES, ids=[c[0] for c in PLAN_CASES])
def test_plan_of_new_geometries(case):
    name, args, geom, kernel = case
    rc, text = _describe(_desc(*args, **geom))
    assert rc == 0, text
    p = _fields(text)
    sh, sw = geom.get("stride_h", 1), geom.get("stride_w", 1)
    dh, dw = geom.get("dil_h", 1), geom.get("dil_w", 1)
    assert p["kernel"] == kernel, p
    bw, bh, bn = (int(v) for v in p["box"].split("x"))
    # the activation box spans bw stride_w x bh stride_h image pixels: a tensor-map box dimension holds at most 256
    assert bw * sw <= 256 and bh * sh <= 256 and bw * bh * bn <= 128, p
    assert p["stride"] == f"{sh}x{sw}" and p["dil"] == f"{dh}x{dw}" and p["group"] == str(geom.get("group", 1))
    if sw != 1 or dw != 1:
        assert p["rowshare"] == "0", p      # neighbouring taps are not neighbouring columns: per-tap delivery
    assert int(p["smem"]) <= 227 * 1024 and int(p["stages"]) >= 2


def test_wide_strided_rows_get_narrower_boxes():
    """Without the 256-element bound a 2048-wide stride-4 layer would take a 128-pixel row box spanning 512 pixels."""
    p = _fields(_describe(_desc(1, 64, 64, 2048, 64, 3, 3, 1, stride_h=4, stride_w=4))[1])
    assert int(p["box"].split("x")[0]) == 64
    p = _fields(_describe(_desc(1, 64, 64, 2048, 64, 3, 3, 1, stride_h=1, stride_w=3))[1])
    assert int(p["box"].split("x")[0]) * 3 <= 256


def test_rowshare_stays_where_the_columns_are_unit_spaced():
    """Stride or dilation in H alone keeps the shared haloed row: only the row coordinate of a tap changes."""
    base = (1, 64, 6, 256, 64, 3, 3, 1)
    assert _fields(_describe(_desc(*base))[1])["rowshare"] == "1"
    assert _fields(_describe(_desc(1, 64, 6, 256, 64, 3, 3, (2, 1), dil_h=2, dil_w=1))[1])["rowshare"] == "1"
    assert _fields(_describe(_desc(1, 64, 6, 256, 64, 3, 3, 2, dil_h=2, dil_w=2))[1])["rowshare"] == "0"
    assert _fields(_describe(_desc(1, 64, 6, 512, 64, 3, 3, 1, stride_h=1, stride_w=2))[1])["rowshare"] == "0"


def test_fused_pool_plan_on_a_strided_layer():
    p = _fields(_describe(_desc(2, 64, 64, 256, 64, 3, 3, 1, pooled_out=True, stride_h=2, stride_w=2))[1])
    bw, bh, _ = (int(v) for v in p["box"].split("x"))
    assert p["pool"] == "1" and bw % 2 == 0 and bh % 2 == 0
    # 33 x 128 -> 17 x 64 outputs: odd height, the epilogue cannot pool
    assert _describe(_desc(2, 64, 33, 128, 64, 3, 3, 1, pooled_out=True, stride_h=2, stride_w=2))[0] == -1


UNSUPPORTED = [
    ("stride5", (1, 64, 32, 32, 64, 3, 3, 1), dict(stride_h=5, stride_w=5)),
    ("stride_negative", (1, 64, 32, 32, 64, 3, 3, 1), dict(stride_h=-1, stride_w=1)),
    ("dil_negative", (1, 64, 32, 32, 64, 3, 3, 1), dict(dil_h=-2, dil_w=1)),
    ("dil_beyond_range", (1, 64, 32, 32, 64, 3, 3, 1), dict(dil_h=1 << 21, dil_w=1)),
    ("dil_beyond_image", (1, 64, 8, 8, 64, 3, 3, 1), dict(dil_h=5, dil_w=5)),
    ("depthwise", (1, 64, 32, 32, 64, 3, 3, 1), dict(group=64)),
    ("group_cin_32", (1, 64, 32, 32, 128, 3, 3, 1), dict(group=2)),
    ("group_cout_32", (1, 128, 32, 32, 64, 3, 3, 1), dict(group=2)),
    ("group_not_dividing", (1, 192, 32, 32, 192, 3, 3, 1), dict(group=2)),
    ("group_negative", (1, 128, 32, 32, 128, 3, 3, 1), dict(group=-2)),
]


@pytest.mark.parametrize("case", UNSUPPORTED, ids=[c[0] for c in UNSUPPORTED])
def test_unsupported_geometries_are_refused(case):
    from mscnn_b200 import capi
    _, args, geom = case
    assert _describe(_desc(*args, **geom))[0] == capi.ERR_INVALID


def test_pool_output_size_rule():
    from mscnn_b200 import capi
    f = capi.lib().mscnn_pool_output_size
    # hand-derived: 7 wide, kernel 3, stride 2, pad 1: ceil(6 / 2) + 1 = 4 windows starting at -1, 1, 3, 5
    assert f(7, 3, 2, 1) == 4
    # 4 wide, kernel 2, stride 2, pad 1: ceil(4 / 2) + 1 = 3, and the third window starts at 3 < 4 + 1: kept
    assert f(4, 2, 2, 1) == 3
    # 3 wide, kernel 2, stride 2, pad 1: ceil(3 / 2) + 1 = 3; the third window would start at column 4 >= 3 + 1: dropped
    assert f(3, 2, 2, 1) == 2
    # 5 wide, kernel 3, stride 3, pad 1: ceil(4 / 3) + 1 = 3; third window starts at 6 - 1 = 5, i.e. (3-1)*3 >= 5 + 1: dropped
    assert f(5, 3, 3, 1) == 2
    for size in range(1, 40):
        for k in range(1, 6):
            for s in range(1, 5):
                for p in range(0, k):
                    if k <= size + 2 * p:
                        assert f(size, k, s, p) == pooled(size, k, s, p), (size, k, s, p)
    assert f(8, 3, 2, 3) == capi.ERR_INVALID and f(8, 0, 1, 0) == capi.ERR_INVALID and f(8, 2, 0, 0) == capi.ERR_INVALID


def test_reference_pool_restatement_hand_cases():
    """AVE divides by the window clipped to the padded extent, not to the image: a constant-2 3x3 map, kernel 3, stride 1,
    pad 1 gives 2 * 4 / 9 in the corners, 2 * 6 / 9 on the edges and 2 in the centre (oracle.port.pool agrees)."""
    from oracle import port
    x = np.full((1, 1, 3, 3), 2.0, dtype=np.float32)
    want = np.array([[8, 12, 8], [12, 18, 12], [8, 12, 8]], dtype=np.float32) / np.float32(9)
    got = pool(x, (3, 3), (1, 1), (1, 1), "AVE")[0, 0]
    assert np.array_equal(got, want) and np.array_equal(port.pool(x, 3, 1, 1, "AVE")[0, 0], want)
    # the window that hangs over the bottom / right edge: clipped to H + pad, so 2 rows x 3 columns = 6 cells, not 9
    x = np.arange(16, dtype=np.float32).reshape(1, 1, 4, 4)
    y = pool(x, (3, 3), (2, 2), (1, 1), "AVE")
    assert y.shape == (1, 1, 3, 3)
    assert y[0, 0, 2, 2] == np.float32(15.0) / np.float32(4)       # window rows 3..5, cols 3..5 clipped to 3..4: 2 x 2 cells
    assert y[0, 0, 0, 0] == np.float32(0 + 1 + 4 + 5) / np.float32(9)
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 3, 9, 14)).astype(np.float32)
    for k, s, p in [(3, 2, 1), (3, 1, 1), (2, 2, 0), (4, 3, 2)]:
        for mode in ("MAX", "AVE"):
            assert np.array_equal(pool(x, (k, k), (s, s), (p, p), mode), port.pool(x, k, s, p, mode)), (k, s, p, mode)


# ---- shapes through a Net (no forward) ----
def _net_text(body, c=64, h=20, w=30):
    return f'input: "d" input_dim: 2 input_dim: {c} input_dim: {h} input_dim: {w}\n' + body


def _conv_layer(param, cout=64):
    return (f'layer {{ name: "c" type: "Convolution" bottom: "d" top: "c" '
            f'convolution_param {{ num_output: {cout} {param} }} }}\n')


def _pool_layer(param):
    return f'layer {{ name: "p" type: "Pooling" bottom: "d" top: "p" pooling_param {{ {param} }} }}\n'


CONV_SHAPES = [
    # prototxt fields, (kh, kw), (pad_h, pad_w), (stride_h, stride_w), (dil_h, dil_w)
    ("kernel_size: 3 pad: 1 stride: 2", (3, 3), (1, 1), (2, 2), (1, 1)),
    ("kernel_size: 3 stride: 3", (3, 3), (0, 0), (3, 3), (1, 1)),
    ("kernel_size: 3 pad: 1 stride_h: 1 stride_w: 2", (3, 3), (1, 1), (1, 2), (1, 1)),
    ("kernel_size: 3 pad: 1 stride: 2 stride: 1", (3, 3), (1, 1), (2, 1), (1, 1)),
    ("kernel_size: 3 pad: 2 dilation: 2", (3, 3), (2, 2), (1, 1), (2, 2)),
    ("kernel_size: 3 pad: 3 dilation: 3 stride: 2", (3, 3), (3, 3), (2, 2), (3, 3)),
    ("kernel_size: 3 pad: 1 dilation: 2 dilation: 1", (3, 3), (1, 1), (1, 1), (2, 1)),
    ("kernel_h: 3 kernel_w: 1 pad_h: 4 pad_w: 0 stride: 4", (3, 1), (4, 0), (4, 4), (1, 1)),
    ("kernel_size: 5 pad: 2 stride: 4", (5, 5), (2, 2), (4, 4), (1, 1)),
]


@pytest.mark.parametrize("hw", [(20, 30), (21, 33), (7, 9)], ids=["even", "odd", "small"])
@pytest.mark.parametrize("case", CONV_SHAPES, ids=[c[0].replace(": ", "").replace(" ", "_") for c in CONV_SHAPES])
def test_convolution_top_shapes(case, hw):
    from mscnn_b200.net import Net
    param, k, pad, stride, dil = case
    h, w = hw
    net = Net(_net_text(_conv_layer(param), h=h, w=w))
    assert net.blob_shape("c") == (2, 64, conv_out(h, k[0], pad[0], stride[0], dil[0]),
                                   conv_out(w, k[1], pad[1], stride[1], dil[1]))
    assert net.param_shapes("c")[0] == (64, 64, k[0], k[1])


def test_grouped_weight_blob_shape():
    from mscnn_b200.net import Net
    for g in (2, 4, 8):
        net = Net(_net_text(_conv_layer(f"kernel_size: 3 pad: 1 group: {g}", cout=512), c=512))
        assert net.param_shapes("c") == [(512, 512 // g, 3, 3), (512,)]
        assert net.blob_shape("c") == (2, 512, 20, 30)
    net = Net(_net_text(_conv_layer("kernel_size: 3 group: 2 stride: 2", cout=256), c=128))
    assert net.param_shapes("c")[0] == (256, 64, 3, 3) and net.blob_shape("c") == (2, 256, 9, 14)


POOL_SHAPES = [
    ("pool: MAX kernel_size: 3 stride: 2 pad: 1", (3, 3), (2, 2), (1, 1)),
    ("pool: AVE kernel_size: 3 stride: 1 pad: 1", (3, 3), (1, 1), (1, 1)),
    ("pool: MAX kernel_h: 3 kernel_w: 2 stride_h: 2 stride_w: 1", (3, 2), (2, 1), (0, 0)),
    ("pool: AVE kernel_h: 3 kernel_w: 2 stride_h: 2 stride_w: 1 pad_h: 1 pad_w: 0", (3, 2), (2, 1), (1, 0)),
    ("pool: MAX kernel_size: 2 stride: 2 pad: 1", (2, 2), (2, 2), (1, 1)),
    ("pool: MAX kernel_size: 3 stride: 3 pad: 1", (3, 3), (3, 3), (1, 1)),
]


@pytest.mark.parametrize("hw", [(20, 30), (21, 33), (3, 5)], ids=["even", "odd", "small"])
@pytest.mark.parametrize("case", POOL_SHAPES, ids=[c[0].replace(": ", "").replace(" ", "_") for c in POOL_SHAPES])
def test_pooling_top_shapes(case, hw):
    """(3, 5) with kernel 2 / stride 2 / pad 1 and kernel 3 / stride 3 / pad 1 are "last window starts in the padding"."""
    from mscnn_b200.net import Net
    param, k, s, p = case
    h, w = hw
    net = Net(_net_text(_pool_layer(param), h=h, w=w))
    assert net.blob_shape("p") == (2, 64, pooled(h, k[0], s[0], p[0]), pooled(w, k[1], s[1], p[1]))
    assert pooled(3, 2, 2, 1) == 2 and pooled(5, 3, 3, 1) == 2      # the decrement cases are among them


def test_global_pooling_follows_the_input_size():
    from mscnn_b200.net import Net
    net = Net(_net_text(_pool_layer("pool: AVE global_pooling: true"), h=24, w=80))
    assert net.blob_shape("p") == (2, 64, 1, 1)
    net.reshape_input("d", 3, 64, 7, 7)
    assert net.blob_shape("p") == (3, 64, 1, 1)


def test_geometry_net_shapes_and_fusion():
    """The end-to-end net of tests/test_conv_geometry_gpu.py: a ReLU folds into every convolution, the 2x2 / 2 MAX pool
    folds into the strided 1x3 convolution, the padded and rectangular pools run themselves."""
    from mscnn_b200.net import Net
    for h, w in GEOMETRY_SIZES:
        net = Net(geometry_net(h, w))
        h1, w1 = conv_out(h, 3, 1, 2), conv_out(w, 3, 1, 2)
        assert net.blob_shape("c_stride2") == (2, 64, h1, w1) and net.blob_shape("c_dil2") == (2, 128, h1, w1)
        assert net.param_shapes("c_group2")[0] == (128, 64, 3, 3)
        h2, w2 = pooled(h1, 3, 2, 1), pooled(w1, 3, 2, 1)
        assert net.blob_shape("p_pad") == (2, 128, h2, w2)
        w3 = conv_out(w2, 3, 1, 2)
        assert net.blob_shape("c_rect") == (2, 64, h2, w3)
        h4, w4 = pooled(h2, 2, 2, 0), pooled(w3, 2, 2, 0)
        assert net.blob_shape("p_fold") == (2, 64, h4, w4)
        assert net.blob_shape("p_rect") == (2, 64, pooled(h4, 3, 2, 1), pooled(w4, 2, 1, 0))
        assert net.blob_shape("p_global") == (2, 64, 1, 1) and net.blob_shape("fc") == (2, 10)
        assert net.fused_producer("p_fold") == "c_rect" and net.fused_producer("relu_c_rect") == "relu_c_rect"
        assert net.fused_producer("p_pad") == "p_pad" and net.fused_producer("p_rect") == "p_rect"
    # the folded pool is computed in the epilogue at the first size (even extents) and by itself at the second
    (ha, wa), (hb, wb) = GEOMETRY_SIZES
    ext = lambda h, w: (pooled(conv_out(h, 3, 1, 2), 3, 2, 1), conv_out(pooled(conv_out(w, 3, 1, 2), 3, 2, 1), 3, 1, 2))
    assert all(v % 2 == 0 for v in ext(ha, wa)) and any(v % 2 for v in ext(hb, wb))


ABORTS = [
    ("depthwise", _net_text(_conv_layer("kernel_size: 3 group: 64")), "multiples of 64"),
    ("group_32_channels", _net_text(_conv_layer("kernel_size: 3 group: 2")), "multiples of 64"),
    ("group_not_dividing", _net_text(_conv_layer("kernel_size: 3 group: 5", cout=65)), "channels_ % group_"),
    ("stride_5", _net_text(_conv_layer("kernel_size: 3 stride: 5")), "strides 1..4"),
    ("dilation_three_times", _net_text(_conv_layer("kernel_size: 3 dilation: 1 dilation: 1 dilation: 1")), "dilation must be"),
    ("pool_pad_not_below_kernel", _net_text(_pool_layer("pool: MAX kernel_size: 2 stride: 2 pad: 2")), "pad_h_ < kernel_h_"),
    ("global_with_kernel", _net_text(_pool_layer("pool: AVE global_pooling: true kernel_size: 3")), "Global_pooling"),
    ("global_with_stride", _net_text(_pool_layer("pool: AVE global_pooling: true stride: 2")), "Global_pooling"),
    ("pool_pad_and_pad_h", _net_text(_pool_layer("pool: MAX kernel_size: 3 pad: 1 pad_h: 1 pad_w: 1")), "pad is pad OR"),
    ("stochastic", _net_text(_pool_layer("pool: STOCHASTIC kernel_size: 2 stride: 2")), "MAX and AVE pooling only"),
]


@pytest.mark.parametrize("case", ABORTS, ids=[c[0] for c in ABORTS])
def test_remaining_checks_abort_with_the_rule(case):
    _, text, message = case
    r = subprocess.run([sys.executable, "-c", "import sys; from mscnn_b200.net import Net; Net(sys.argv[1])", text],
                       capture_output=True, text=True, cwd=str(ROOT))
    assert r.returncode != 0 and message in r.stderr, r.stderr[-600:]


# ---- the test references against the reference's own layers ----
def _ref_single_layer(text, x, weights=None, top="c"):
    from oracle import ref
    net = ref.RefNet(text)
    if weights:
        net.set_params(weights)
    net.set_blob("d", x)
    net.forward()
    return net.blob(top)


@pytest.fixture(scope="module")
def ref_built():
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref is not built (needs the reference sources)")


REF_CONVS = [("kernel_size: 3 pad: 1 stride: 2", 1), ("kernel_size: 3 pad: 2 dilation: 2", 1),
             ("kernel_size: 3 pad: 3 dilation: 3 stride: 2", 1), ("kernel_size: 3 pad: 1 dilation: 2 dilation: 1", 1),
             ("kernel_size: 3 pad: 1 stride_h: 1 stride_w: 2", 1), ("kernel_size: 3 pad: 1 group: 2 stride: 2", 2),
             ("kernel_h: 3 kernel_w: 1 pad_h: 4 pad_w: 0 stride: 3", 1)]


@pytest.mark.parametrize("case", REF_CONVS, ids=[c[0].replace(": ", "").replace(" ", "_") for c in REF_CONVS])
def test_torch_fp64_convolution_matches_the_reference_layer(ref_built, case):
    """The GPU tests compare with torch's fp64 convolution; here that reference is held to ConvolutionLayer::Forward_cpu
    (fp32 im2col + sgemm: 1e-4 of the output's rms, the reference's own test tolerance)."""
    import torch
    import torch.nn.functional as F
    param, group = case
    rng = np.random.default_rng(11)
    x = rng.standard_normal((2, 8, 13, 18)).astype(np.float32)
    text = _net_text(_conv_layer(param, cout=6), c=8, h=13, w=18)
    geom = next(c for c in CONV_SHAPES + [("kernel_size: 3 pad: 1 group: 2 stride: 2", (3, 3), (1, 1), (2, 2), (1, 1)),
                                          ("kernel_h: 3 kernel_w: 1 pad_h: 4 pad_w: 0 stride: 3", (3, 1), (4, 0), (3, 3), (1, 1))]
                if c[0] == param)
    w = (rng.standard_normal((6, 8 // group) + geom[1]) * 0.2).astype(np.float32)
    b = rng.standard_normal(6).astype(np.float32)
    got = _ref_single_layer(text, x, {"c": [w, b]})
    want = F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(),
                    stride=geom[3], padding=geom[2], dilation=geom[4], groups=group).numpy()
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-4 * np.sqrt((want ** 2).mean())


@pytest.mark.parametrize("mode", ["MAX", "AVE"])
@pytest.mark.parametrize("case", POOL_SHAPES, ids=[c[0].replace(": ", "").replace(" ", "_") for c in POOL_SHAPES])
def test_pool_restatement_matches_the_reference_layer(ref_built, case, mode):
    param, k, s, p = case
    param = re.sub(r"pool: \w+", f"pool: {mode}", param)
    rng = np.random.default_rng(12)
    for h, w in [(9, 14), (3, 5), (12, 7)]:
        x = rng.standard_normal((2, 4, h, w)).astype(np.float32)
        got = _ref_single_layer(_net_text(_pool_layer(param), c=4, h=h, w=w), x, top="p")
        assert np.array_equal(got, pool(x, k, s, p, mode)), (h, w)


def test_global_pool_restatement_matches_the_reference_layer(ref_built):
    rng = np.random.default_rng(13)
    x = rng.standard_normal((2, 4, 7, 9)).astype(np.float32)
    for mode in ("MAX", "AVE"):
        got = _ref_single_layer(_net_text(_pool_layer(f"pool: {mode} global_pooling: true"), c=4, h=7, w=9), x, top="p")
        assert np.array_equal(got, pool(x, (7, 9), (1, 1), (0, 0), mode))
