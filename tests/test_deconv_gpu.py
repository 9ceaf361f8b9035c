"""Deconvolution on the device: mscnn_deconv_forward (dense and 64-aligned grouped layers, by output phase on the
implicit-GEMM kernel) and mscnn_deconv_depthwise_forward against torch's fp64 conv_transpose2d (held to the reference's
own layer in tests/test_deconv_cpu.py; tolerances of tests/test_conv_geometry_gpu.py), the exact identities between a
phase and mscnn_conv_forward on its sub-kernel, and one net with every served geometry against the reference's own
layers (fixture tests/golden/deconv_net.npz, made by tests/golden/make_deconv_golden.py)."""
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from deconv_ref import DECONV_BLOBS, DECONV_CONCATS, DECONV_SIZES, axis_phase, deconv_net, deconv_out, phase_kernel

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "deconv_net.npz"


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _operands(cuda, n, cin, h, w, cout, k, group=1, seed=1706):
    kh, kw = _pair(k)
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn((n, cin, h, w), generator=g).to(cuda)
    wt = (torch.randn((cin, cout // group, kh, kw), generator=g) * (2.0 / (cin // group * kh * kw)) ** 0.5).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    return x, wt, b


def _ref(x, wt, b, stride, pad, dil, group, relu=False):
    y = F.conv_transpose2d(x.double(), wt.double(), None if b is None else b.double(), stride=_pair(stride),
                           padding=_pair(pad), dilation=_pair(dil), groups=group)
    return torch.relu(y) if relu else y


def _check(name, got, ref, split):
    rms = float(ref.pow(2).mean().sqrt())
    tol_rel, tol_abs = (1e-4, 1e-4 * rms) if split else (2.0 ** -8, 1e-5 * rms)
    err = (got.double() - ref).abs()
    bad = err > tol_rel * ref.abs() + tol_abs
    if bad.any():
        idx = bad.nonzero()
        pytest.fail(f"{name}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float(err.max()):.3e}, ref rms "
                    f"{rms:.3e}; first bad (n, c, h, w) {idx[:6].tolist()}; distinct bad h {idx[:, 2].unique()[:12].tolist()} "
                    f"w {idx[:, 3].unique()[:12].tolist()} c {idx[:, 1].unique()[:8].tolist()}")


CASES = [
    # name,          N, Cin, H,  W, Cout, k,   stride, pad, dil, group
    ("k4s2p1",       1, 64, 12, 20, 64, 4, 2, 1, 1, 1),
    ("k4s2p1_512",   1, 512, 6, 10, 512, 4, 2, 1, 1, 1),       # BLOCK_N 256
    ("k2s2",         2, 128, 9, 13, 128, 2, 2, 0, 1, 1),       # BLOCK_N 128
    ("k3s2p1_odd",   3, 64, 7, 11, 64, 3, 2, 1, 1, 1),         # odd output extent
    ("k1s1",         1, 64, 8, 8, 64, 1, 1, 0, 1, 1),
    ("k3s1p1",       2, 64, 10, 16, 64, 3, 1, 1, 1, 1),
    ("k5s3p2",       1, 64, 9, 10, 64, 5, 3, 2, 1, 1),
    ("k6s4p1",       1, 64, 7, 9, 128, 6, 4, 1, 1, 1),
    ("k7s4p3",       2, 64, 5, 6, 64, 7, 4, 3, 1, 1),
    ("k8s8",         1, 64, 4, 5, 64, 8, 8, 0, 1, 1),
    ("k8s4p2",       1, 64, 6, 7, 64, 8, 4, 2, 1, 1),
    ("k16s8p4",      1, 64, 3, 4, 64, 16, 8, 4, 1, 1),
    ("k1s4_tapless", 1, 64, 5, 7, 24, 1, 4, 0, 1, 1),         # k < s: 15 of 16 phases hold the bias; Cout 24
    ("k2s3",         1, 64, 6, 6, 64, 2, 3, 0, 1, 1),
    ("k3s2p2d2",     2, 64, 6, 9, 64, 3, 2, 2, 2, 1),         # gcd(s, d) = 2: the odd phases have no tap
    ("k3s1p3d3",     1, 64, 8, 9, 64, 3, 1, 3, 3, 1),
    ("k3s2p0d3",     1, 64, 6, 7, 64, 3, 2, 0, 3, 1),
    ("k4s2p3",       1, 64, 6, 8, 64, 4, 2, 3, 1, 1),         # p > d (k - 1) / 2: negative sub-pads
    ("k6s2p6",       1, 64, 8, 132, 64, 6, 2, 6, 1, 1),       # pad -1 with the shared haloed row
    ("rect",         2, 64, 7, 9, 64, (3, 5), (2, 3), (1, 0), (1, 2), 1),
    ("rect_s1x4",    1, 64, 5, 6, 64, (2, 4), (1, 4), (0, 1), 1, 1),
    ("g2_s2",        1, 128, 6, 10, 128, 4, 2, 1, 1, 2),
    ("g4_512",       1, 512, 5, 6, 512, 2, 2, 0, 1, 4),
    ("g2_rect",      2, 256, 5, 7, 128, (3, 2), (2, 1), (1, 0), (2, 1), 2),
    ("cout24_n3",    3, 64, 5, 9, 24, 3, 2, 1, 1, 1),
    ("many_tiles",   4, 128, 64, 96, 128, 4, 2, 1, 1, 1),     # 192 tiles per phase: more than SMs
    ("wide",         1, 64, 4, 300, 64, 3, 2, 1, 1, 1),       # output rows of 599 pixels
]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_deconv_parity(cuda, case, split):
    from mscnn_b200 import ops
    name, n, cin, h, w, cout, k, stride, pad, dil, group = case
    x, wt, b = _operands(cuda, n, cin, h, w, cout, k, group)
    xp = ops.nchw_to_planes(x, split)
    wp = ops.pack_deconv_weights(wt, b, split, stride, pad, dil, group)
    got = ops.planes_to_nchw(ops.deconv_forward(xp, wp, relu=True))
    torch.cuda.synchronize()
    src = (x, wt) if split else (x.bfloat16().float(), wt.bfloat16().float())
    ref = _ref(*src, b, stride, pad, dil, group, relu=True)
    assert tuple(got.shape) == tuple(ref.shape)
    _check(name, got, ref, split)


@pytest.mark.parametrize("no_fat", [False, True], ids=["fat", "term_major"])
@pytest.mark.parametrize("case", [c for c in CASES if c[0] in ("k4s2p1", "k3s2p1_odd", "k3s2p2d2", "rect", "g2_s2",
                                                                "k6s2p6", "cout24_n3")], ids=lambda c: c[0])
def test_deconv_both_operand_orders(cuda, case, no_fat, monkeypatch):
    from mscnn_b200 import ops
    name, n, cin, h, w, cout, k, stride, pad, dil, group = case
    x, wt, b = _operands(cuda, n, cin, h, w, cout, k, group, seed=1707)
    xp = ops.nchw_to_planes(x, True)
    try:
        if no_fat:
            monkeypatch.setenv("MSCNN_NO_FAT", "1")
        ops.reload_config()
        wp = ops.pack_deconv_weights(wt, b, True, stride, pad, dil, group)
        got = ops.planes_to_nchw(ops.deconv_forward(xp, wp))
        torch.cuda.synchronize()
    finally:
        monkeypatch.delenv("MSCNN_NO_FAT", raising=False)
        ops.reload_config()
    _check(name, got, _ref(x, wt, b, stride, pad, dil, group), True)


# ---- exact identities ----
def _sub_conv(ops, xp, wt, b, split, taps_h, taps_w, pad, dil, group):
    """mscnn_conv_forward on one phase's sub-kernel (channel axes swapped, taps reversed), packed by
    mscnn_pack_conv_weights."""
    wsub = torch.from_numpy(np.ascontiguousarray(phase_kernel(wt.cpu().numpy(), taps_h, taps_w, group))).to(wt.device)
    return ops.planes_to_nchw(ops.conv_forward(xp, ops.pack_conv_weights(wsub, b, split), pad, relu=True, dilation=dil,
                                               group=group))


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", [(2, 64, 9, 14, 64, 3, 1, 1), (1, 128, 6, 20, 256, (3, 5), (1, 2), 2),
                                  (1, 64, 4, 128, 64, 3, 1, 1), (1, 512, 5, 6, 512, 2, 1, 1)],
                         ids=["k3p1", "rect_dil", "k3p1_rowshare", "k2p1_512"])
def test_stride1_deconv_equals_the_flipped_convolution_bitwise(cuda, case, split):
    """Stride 1 has one phase: the convolution with the transposed, reversed kernel and pad d (k - 1) - p >= 0."""
    from mscnn_b200 import ops
    n, cin, h, w, cout, k, pad, dil = case
    (kh, kw), (ph, pw), (dh, dw) = _pair(k), _pair(pad), _pair(dil)
    x, wt, b = _operands(cuda, n, cin, h, w, cout, k, seed=31)
    xp = ops.nchw_to_planes(x, split)
    got = ops.planes_to_nchw(ops.deconv_forward(xp, ops.pack_deconv_weights(wt, b, split, 1, pad, dil), relu=True))
    want = _sub_conv(ops, xp, wt, b, split, list(range(kh)), list(range(kw)), (dh * (kh - 1) - ph, dw * (kw - 1) - pw),
                     (dh, dw), 1)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", [(2, 64, 7, 10, 64, 4, 2, 1, 1, 1), (1, 128, 6, 9, 128, (5, 3), (3, 2), (1, 0), 1, 2),
                                  (1, 64, 4, 128, 64, 6, 2, 2, 1, 1), (1, 256, 5, 6, 256, 4, 4, 0, (1, 2), 1)],
                         ids=["k4s2p1", "g2_rect", "k6s2p2_rowshare", "k4s4_dil"])
def test_each_phase_equals_its_sub_convolution_bitwise(cuda, case, split):
    """Phase (r_h, r_w), read out of the output with [r_h::s_h, r_w::s_w], is mscnn_conv_forward of its sub-kernel with
    the sub-dilation and the (here non-negative) sub-pad: same kernel instantiation, box and summation order."""
    from mscnn_b200 import ops
    n, cin, h, w, cout, k, stride, pad, dil, group = case
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = _pair(k), _pair(stride), _pair(pad), _pair(dil)
    x, wt, b = _operands(cuda, n, cin, h, w, cout, k, group, seed=32)
    xp = ops.nchw_to_planes(x, split)
    got = ops.planes_to_nchw(ops.deconv_forward(xp, ops.pack_deconv_weights(wt, b, split, stride, pad, dil, group),
                                                relu=True))
    ho, wo = got.shape[2:]
    checked = 0
    for rh in range(sh):
        th, dil_h, pad_h, qh = axis_phase(kh, sh, ph, dh, ho, rh)
        for rw in range(sw):
            tw, dil_w, pad_w, qw = axis_phase(kw, sw, pw, dw, wo, rw)
            if not th or not tw or pad_h < 0 or pad_w < 0:
                continue
            want = _sub_conv(ops, xp, wt, b, split, th, tw, (pad_h, pad_w), (dil_h, dil_w), group)
            torch.cuda.synchronize()
            # where the phase extends past the convolution's own extent it reads zeros beyond the input: compare the
            # outputs both have
            mh, mw = min(qh, want.shape[2]), min(qw, want.shape[3])
            assert mh > 0 and mw > 0
            assert torch.equal(got[:, :, rh::sh, rw::sw][:, :, :mh, :mw], want[:, :, :mh, :mw]), (rh, rw)
            checked += 1
    assert checked >= 1


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_tapless_phases_hold_exactly_the_bias(cuda, split):
    from mscnn_b200 import ops
    for k, stride, pad, dil in [(1, 4, 0, 1), (3, 2, 2, 2), (2, 3, 0, 3)]:
        x, wt, b = _operands(cuda, 2, 64, 5, 7, 128, k, seed=33)
        xp = ops.nchw_to_planes(x, split)
        out = ops.deconv_forward(xp, ops.pack_deconv_weights(wt, b, split, stride, pad, dil))
        torch.cuda.synchronize()
        got = out.float()
        ho, wo = got.shape[1:3]
        bias = b.bfloat16().float() if not split else (b.bfloat16().float() + (b - b.bfloat16().float()).bfloat16().float())
        tapless = 0
        for rh in range(stride):
            for rw in range(stride):
                th, _, _, qh = axis_phase(k, stride, pad, dil, ho, rh)
                tw, _, _, qw = axis_phase(k, stride, pad, dil, wo, rw)
                if qh and qw and (not th or not tw):
                    assert torch.equal(got[:, rh::stride, rw::stride], bias.expand(2, qh, qw, 128)), (k, stride, rh, rw)
                    tapless += 1
        assert tapless > 0


def test_unserved_geometry_is_an_error_and_writes_nothing(cuda):
    from mscnn_b200 import capi, ops
    x, wt, b = _operands(cuda, 1, 128, 6, 6, 128, 4, seed=34)
    xp = ops.nchw_to_planes(x, True)
    wp = ops.pack_deconv_weights(wt, b, True, 2, 1)
    out = ops.Planes(torch.full((1, 12, 12, 128), 7.0, dtype=torch.bfloat16, device=cuda),
                     torch.full((1, 12, 12, 128), 7.0, dtype=torch.bfloat16, device=cuda), 128)
    for field, value in [("stride_h", 9), ("group", 4), ("dyn_n", out.hi.data_ptr())]:
        d = ops.deconv_desc(xp, wp)
        d.y_hi, d.y_lo = out.hi.data_ptr(), out.lo.data_ptr()
        setattr(d, field, value)
        assert capi.lib().mscnn_deconv_forward(d, torch.cuda.current_stream().cuda_stream) == capi.ERR_INVALID, field
    torch.cuda.synchronize()
    assert bool((out.hi == 7.0).all()) and bool((out.lo == 7.0).all())


# ---- depthwise ----
DW_CASES = [
    # name, C, H, W, k, stride, pad, dil
    ("bilinear_2x", 512, 12, 20, 4, 2, 1, 1),
    ("bilinear_4x", 64, 9, 11, 8, 4, 2, 1),
    ("bilinear_8x", 512, 5, 6, 16, 8, 4, 1),
    ("k2s2", 64, 7, 9, 2, 2, 0, 1),
    ("k3s1p1", 72, 6, 7, 3, 1, 1, 1),
    ("k5s3p1", 64, 6, 5, 5, 3, 1, 1),
    ("k3s2p2d2", 64, 6, 7, 3, 2, 2, 2),
    ("k3s1p0d3", 64, 5, 6, 3, 1, 0, 3),
    ("rect", 64, 6, 7, (3, 6), (2, 4), (1, 2), (2, 1)),
    ("k1s8", 64, 4, 3, 1, 8, 0, 1),
    ("k12s6p3", 128, 4, 5, 12, 6, 3, 1),
]


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", DW_CASES, ids=[c[0] for c in DW_CASES])
def test_depthwise_parity(cuda, case, split, bias):
    from mscnn_b200 import ops
    name, c, h, w, k, stride, pad, dil = case
    g = torch.Generator(device="cpu").manual_seed(41)
    x = torch.randn((2, c, h, w), generator=g).to(cuda)
    wt = torch.randn((c, 1) + _pair(k), generator=g).to(cuda)
    b = torch.randn((c,), generator=g).to(cuda) if bias else None
    out = ops.deconv_depthwise_forward(ops.nchw_to_planes(x, split), wt, b, stride, pad, dil)
    got = ops.planes_to_nchw(out)
    torch.cuda.synchronize()
    src = (x, wt) if split else (x.bfloat16().float(), wt)
    ref = _ref(*src, b, stride, pad, dil, c)
    assert tuple(got.shape) == tuple(ref.shape)
    _check(name, got, ref, split)


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_deconv2x_entry_is_the_depthwise_4_2_1_layer_bitwise(cuda, split):
    from mscnn_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(42)
    x = torch.randn((2, 512, 11, 17), generator=g).to(cuda)
    wt = torch.randn((512, 1, 4, 4), generator=g).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    a = ops.deconv2x_forward(xp, wt)
    b = ops.deconv_depthwise_forward(xp, wt, None, 2, 1)
    torch.cuda.synchronize()
    assert torch.equal(a.hi, b.hi) and (not split or torch.equal(a.lo, b.lo))


# ---- one net with every served geometry, against the reference's own layers ----
@pytest.fixture()
def side_stream(cuda):
    from mscnn_b200 import net as mnet
    s = torch.cuda.Stream()
    prev = torch.cuda.current_stream()
    torch.cuda.set_stream(s)
    mnet.set_stream(s.cuda_stream)
    yield s
    torch.cuda.synchronize()
    torch.cuda.set_stream(prev)
    mnet.set_stream(prev.cuda_stream)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_deconv_net_matches_the_reference_layers(side_stream, graph):
    """Blob by blob within the 1e-3 gate of the fp32-faithful mode, at two input sizes with a reshape_input in between;
    the Concat tops against the concatenation of their parts."""
    from mscnn_b200 import net as mnet, synth
    mnet.set_precision("fp32")
    golden = np.load(GOLDEN)
    h0, w0 = DECONV_SIZES[0]
    net = mnet.Net(deconv_net(h0, w0))
    net.set_params(synth.make_weights(net.layers()))
    net.set_graph(graph)
    replays = 0
    for h, w in DECONV_SIZES + DECONV_SIZES[:1]:
        net.reshape_input("data", 2, 3, h, w)
        for _ in range(3 if graph else 1):
            net.forward(data=synth.make_images(2, h, w))
            replays += int(net.graph_replayed())
        wants = {name: golden[f"{h}x{w}/{name}"] for name in DECONV_BLOBS}
        wants.update({cat: np.concatenate([wants[a], wants[b]], axis=1) for cat, (a, b) in DECONV_CONCATS.items()})
        for name, want in wants.items():
            got = net.blob(name).reshape(want.shape)
            err = float(np.abs(got - want).max()) / float(np.sqrt((want.astype(np.float64) ** 2).mean()))
            assert err <= 1e-3, (h, w, name, err)
    assert replays >= (3 if graph else 0) and (graph or replays == 0)
