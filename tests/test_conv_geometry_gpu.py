"""Convolution with stride, dilation and groups, and pooling with padding, rectangular windows and global pooling, on
the device: mscnn_conv_forward against the fp64 convolution of the same operands (tolerances of tests/test_conv_gpu.py),
the exact identities that pin the group offsets and the strided coordinates, mscnn_pool2d_forward_dyn against the
restated reference pooling, and one small net with every new geometry against the reference's own layers (fixture
tests/golden/geometry_net.npz, made by tests/golden/make_geometry_golden.py)."""
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conv_geometry_ref import GEOMETRY_BLOBS, GEOMETRY_SIZES, geometry_net, pool

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "geometry_net.npz"


def _pair(v):
    return (v, v) if isinstance(v, int) else v


def _operands(cuda, n, cin, h, w, cout, k, group=1, seed=1706):
    kh, kw = _pair(k)
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn((n, cin, h, w), generator=g).to(cuda)
    wt = (torch.randn((cout, cin // group, kh, kw), generator=g) * (2.0 * group / (cin * kh * kw)) ** 0.5).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    return x, wt, b


def _ref_conv(x, w, b, pad, stride, dil, group, relu):
    y = F.conv2d(x.double(), w.double(), b.double(), stride=_pair(stride), padding=_pair(pad), dilation=_pair(dil),
                 groups=group)
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
    # name,          N, Cin, H,  W, Cout, k,   pad,    stride, dil,  group
    ("s2",           1, 64, 16, 32, 64, 3, 1, 2, 1, 1),
    ("s2_odd",       3, 64, 9, 31, 64, 3, 1, 2, 1, 1),
    ("s1x2",         2, 64, 12, 40, 128, 3, 1, (1, 2), 1, 1),
    ("s2x1",         2, 64, 12, 40, 128, 3, 1, (2, 1), 1, 1),
    ("s3",           1, 128, 25, 31, 256, 3, 1, 3, 1, 1),
    ("s4_k5",        1, 64, 37, 50, 64, 5, 2, 4, 1, 1),
    ("s4_n32",       3, 64, 21, 19, 24, 3, 1, 4, 1, 1),
    ("s2_k1",        2, 64, 9, 24, 64, 1, 0, 2, 1, 1),
    ("s2_k3x1",      1, 64, 11, 20, 64, (3, 1), (1, 0), 2, 1, 1),
    # the last strided column / row reads the padding only: W + pad - 1 is a tap start (W = 8, stride 2, pad 2, k = 1)
    ("s2_lastcol_in_pad", 1, 64, 8, 8, 64, 1, 2, 2, 1, 1),
    ("s2_pad_beyond_reach", 1, 64, 10, 14, 64, 3, 3, 2, 1, 1),
    ("s2_tiny",      1, 64, 3, 5, 64, 3, 1, 2, 1, 1),
    ("s2_wide",      1, 64, 4, 1030, 64, 3, 1, 2, 1, 1),           # more than one box per row, 128-pixel boxes spanning 256
    ("s4_wide",      1, 64, 8, 1100, 64, 3, 1, 4, 1, 1),           # boxes bounded to 64 pixels
    ("s2_many",      2, 64, 128, 320, 128, 3, 1, 2, 1, 1),         # more tiles than SMs
    ("s2_bn256_2nt", 1, 128, 16, 48, 512, 3, 1, 2, 1, 1),
    ("d2",           1, 64, 16, 32, 64, 3, 2, 1, 2, 1),
    ("d3",           2, 64, 13, 29, 128, 3, 3, 1, 3, 1),
    ("d2x1",         1, 64, 12, 256, 64, 3, (2, 1), 1, (2, 1), 1),  # shared haloed row with dilated rows
    ("d2_w256",      1, 64, 6, 256, 64, 3, 2, 1, 2, 1),
    ("d2_bn256",     1, 256, 12, 40, 256, 3, 2, 1, 2, 1),
    ("d2_pad0",      1, 64, 12, 20, 64, 3, 0, 1, 2, 1),
    ("d2_k5",        1, 64, 20, 24, 64, 5, 4, 1, 2, 1),
    ("s2_d2",        2, 128, 24, 40, 128, 3, 2, 2, 2, 1),
    ("s2_d2_n32",    1, 64, 17, 23, 9, 3, 2, 2, 2, 1),
    ("g2_512",       1, 512, 6, 20, 512, 3, 1, 1, 1, 2),
    ("g4_512",       1, 512, 6, 20, 512, 3, 1, 1, 1, 4),
    ("g8_512",       3, 512, 5, 9, 512, 3, 1, 1, 1, 8),
    ("g2_128_256",   1, 128, 12, 40, 256, 3, 1, 1, 1, 2),
    ("g2_w128",      1, 128, 4, 256, 128, 3, 1, 1, 1, 2),          # grouped with the shared haloed row
    ("g4_s2_d2",     2, 256, 18, 26, 256, 3, 2, 2, 2, 4),
    ("g2_k1",        1, 128, 8, 24, 128, 1, 0, 1, 1, 2),
]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_geometry_planes(cuda, case, split):
    from mscnn_b200 import ops
    name, n, cin, h, w, cout, k, pad, stride, dil, group = case
    x, wt, b = _operands(cuda, n, cin, h, w, cout, k, group)
    xp = ops.nchw_to_planes(x, split)
    wp = ops.pack_conv_weights(wt, b, split)
    if cout > 32:
        got = ops.planes_to_nchw(ops.conv_forward(xp, wp, pad, relu=True, stride=stride, dilation=dil, group=group))
    else:
        got = ops.conv_forward(xp, wp, pad, relu=True, out_f32=True, stride=stride, dilation=dil, group=group)
    torch.cuda.synchronize()
    if split:
        ref = _ref_conv(x, wt, b, pad, stride, dil, group, True)
    else:
        ref = _ref_conv(x.bfloat16().float(), wt.bfloat16().float(), b, pad, stride, dil, group, True)
    assert tuple(got.shape) == tuple(ref.shape)
    _check(name, got, ref, split)


@pytest.mark.parametrize("no_fat", [False, True], ids=["fat", "term_major"])
@pytest.mark.parametrize("case", [c for c in CASES if c[0] in ("s2_odd", "s1x2", "d3", "s2_d2", "g4_512", "g2_128_256")],
                         ids=lambda c: c[0])
def test_conv_geometry_both_operand_orders(cuda, case, no_fat, monkeypatch):
    """BLOCK_N <= 128 layers of the split path in fat stages and, with MSCNN_NO_FAT, in the term-major order BLOCK_N = 256
    always takes: both within tolerance of the fp64 convolution."""
    from mscnn_b200 import ops
    name, n, cin, h, w, cout, k, pad, stride, dil, group = case
    x, wt, b = _operands(cuda, n, cin, h, w, cout, k, group, seed=1707)
    xp, wp = ops.nchw_to_planes(x, True), ops.pack_conv_weights(wt, b, True)
    try:
        if no_fat:
            monkeypatch.setenv("MSCNN_NO_FAT", "1")
        ops.reload_config()
        got = ops.planes_to_nchw(ops.conv_forward(xp, wp, pad, relu=False, stride=stride, dilation=dil, group=group))
        torch.cuda.synchronize()
    finally:
        monkeypatch.delenv("MSCNN_NO_FAT", raising=False)
        ops.reload_config()
    _check(name, got, _ref_conv(x, wt, b, pad, stride, dil, group, False), True)


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("mode", ["nchw_f32", "nhwc_f32"])
def test_conv_geometry_fp32_output_modes(cuda, mode, split):
    from mscnn_b200 import capi, ops
    x, wt, b = _operands(cuda, 2, 64, 15, 22, 64, 3, seed=3)
    xp, wp = ops.nchw_to_planes(x, split), ops.pack_conv_weights(wt, b, split)
    kw = dict(stride=2, dilation=(2, 1))
    if mode == "nchw_f32":
        got = ops.conv_forward(xp, wp, (2, 1), relu=False, out_f32=True, **kw)
    else:
        got = ops.conv_forward(xp, wp, (2, 1), relu=False, out_mode=capi.OUT_NHWC_F32, **kw).permute(0, 3, 1, 2)[:, :64]
    torch.cuda.synchronize()
    src = (x, wt) if split else (x.bfloat16().float(), wt.bfloat16().float())
    ref = _ref_conv(*src, b, (2, 1), 2, (2, 1), 1, False)
    rms = float(ref.pow(2).mean().sqrt())
    assert float((got.double() - ref).abs().max()) <= (1e-4 if split else 1e-5) * 2 * rms


@pytest.mark.parametrize("group", [2, 4, 8])
@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_grouped_equals_ungrouped_slices_bitwise(cuda, group, split):
    """A grouped convolution is, bit for bit, the g ungrouped convolutions of the channel slices: the same kernel
    instantiation, box and summation order, so any difference is a wrong group offset."""
    from mscnn_b200 import ops
    cin = cout = 512
    x, wt, b = _operands(cuda, 2, cin, 7, 18, cout, 3, group, seed=9)
    xp, wp = ops.nchw_to_planes(x, split), ops.pack_conv_weights(wt, b, split)
    got = ops.planes_to_nchw(ops.conv_forward(xp, wp, 1, relu=True, stride=(1, 2), group=group))
    cg, og = cin // group, cout // group
    for k in range(group):
        xs = ops.nchw_to_planes(x[:, k * cg:(k + 1) * cg].contiguous(), split)
        ws = ops.pack_conv_weights(wt[k * og:(k + 1) * og].contiguous(), b[k * og:(k + 1) * og].contiguous(), split)
        part = ops.planes_to_nchw(ops.conv_forward(xs, ws, 1, relu=True, stride=(1, 2)))
        torch.cuda.synchronize()
        assert torch.equal(got[:, k * og:(k + 1) * og], part), k


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("s", [2, 3, 4])
def test_strided_equals_subsampled_stride1_bitwise(cuda, s, split, monkeypatch):
    """Stride s reads the taps of every s-th stride-1 output in the same (dy, chunk, dx) order: with per-tap delivery on
    both sides (MSCNN_NO_ROWSHARE) and the same BLOCK_N the results are the same bits."""
    from mscnn_b200 import ops
    x, wt, b = _operands(cuda, 2, 128, 17, 41, 128, 3, seed=4)
    xp, wp = ops.nchw_to_planes(x, split), ops.pack_conv_weights(wt, b, split)
    try:
        monkeypatch.setenv("MSCNN_NO_ROWSHARE", "1")
        ops.reload_config()
        full = ops.planes_to_nchw(ops.conv_forward(xp, wp, 1, relu=True))
        strided = ops.planes_to_nchw(ops.conv_forward(xp, wp, 1, relu=True, stride=s))
        torch.cuda.synchronize()
    finally:
        monkeypatch.delenv("MSCNN_NO_ROWSHARE", raising=False)
        ops.reload_config()
    assert torch.equal(strided, full[:, :, ::s, ::s].contiguous())


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", [(2, 64, 32, 48, 64, 2, 1, 1), (1, 128, 28, 44, 128, 1, 2, 2), (2, 128, 16, 72, 128, (1, 2), 1, 2),
                                  (1, 64, 20, 512, 64, (1, 2), 1, 1)],
                         ids=["s2", "d2_g2", "s1x2_g2", "s1x2_w256"])
def test_fused_pool_on_new_geometries_bitwise(cuda, case, split):
    """The 2x2 / 2 MAX pool in the epilogue of a strided / dilated / grouped layer == the un-fused layer followed by
    mscnn_pool_forward, bit for bit; the pool-only form gives the same pooled planes."""
    from mscnn_b200 import ops
    n, cin, h, w, cout, stride, dil, group = case
    x, wt, b = _operands(cuda, n, cin, h, w, cout, 3, group, seed=21)
    xp, wp = ops.nchw_to_planes(x, split), ops.pack_conv_weights(wt, b, split)
    kw = dict(stride=stride, dilation=dil, group=group)
    y_ref = ops.conv_forward(xp, wp, dil, relu=True, **kw)
    assert y_ref.shape[1] % 2 == 0 and y_ref.shape[2] % 2 == 0
    p_ref = ops.pool_forward(y_ref, 2, 2)
    y_both, p_both = ops.conv_forward(xp, wp, dil, relu=True, pool="both", **kw)
    p_only = ops.conv_forward(xp, wp, dil, relu=True, pool="only", **kw)
    torch.cuda.synchronize()
    assert torch.equal(y_both.hi, y_ref.hi)
    for cand in (p_both, p_only):
        assert torch.equal(cand.hi, p_ref.hi) and (not split or torch.equal(cand.lo, p_ref.lo))


def test_dyn_n_leaves_the_remaining_rows_untouched(cuda):
    """A device count below N: the images below it equal the launch without a count, and nothing is written from the
    end of the last box of box_n images that holds one of them."""
    from mscnn_b200 import ops
    x, wt, b = _operands(cuda, 5, 128, 45, 60, 128, 3, 2, seed=6)
    xp, wp = ops.nchw_to_planes(x, True), ops.pack_conv_weights(wt, b, True)
    kw = dict(stride=2, dilation=2, group=2)
    full = ops.conv_forward(xp, wp, 2, relu=True, **kw)
    assert full.shape[1:3] == (23, 30)          # tiled in 30x4x1 boxes: a box never spans two images
    for count in (0, 2, 5, 9):
        out = ops.Planes(torch.full_like(full.hi, 7.0), torch.full_like(full.lo, 7.0), full.channels)
        dyn = torch.tensor([count], dtype=torch.int32, device=cuda)
        ops.conv_forward(xp, wp, 2, relu=True, dyn=dyn, out=out, **kw)
        torch.cuda.synchronize()
        k = min(count, 5)
        assert torch.equal(out.hi[:k], full.hi[:k]) and torch.equal(out.lo[:k], full.lo[:k])
        assert bool((out.hi[k:] == 7.0).all()) and bool((out.lo[k:] == 7.0).all())


def test_unserved_geometry_is_an_error_not_a_result(cuda):
    from mscnn_b200 import capi, ops
    x, wt, b = _operands(cuda, 1, 64, 12, 12, 64, 3)
    xp, wp = ops.nchw_to_planes(x, True), ops.pack_conv_weights(wt, b, True)
    with pytest.raises(capi.MscnnError):
        ops.conv_forward(xp, wp, 1, relu=False, stride=5)


# ---- pooling ----
def _bf16_exact(a):
    return torch.from_numpy(a).bfloat16().float().numpy()


POOLS = [
    # name, H, W, kernel, stride, pad
    ("k3s2p1", 24, 80, 3, 2, 1), ("k3s2p1_odd", 9, 15, 3, 2, 1), ("k3s1p1", 7, 9, 3, 1, 1),
    ("k3x2_s2x1", 12, 16, (3, 2), (2, 1), 0), ("k3x2_s2x1_p1x0", 11, 13, (3, 2), (2, 1), (1, 0)),
    ("k2s2p1_decrement", 3, 5, 2, 2, 1), ("k3s3p1_decrement", 5, 8, 3, 3, 1), ("k2x3_p0x2", 8, 8, (2, 3), (2, 2), (0, 2)),
]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("mode", ["MAX", "AVE"])
@pytest.mark.parametrize("case", POOLS, ids=[c[0] for c in POOLS])
def test_pool_geometry_parity(cuda, case, mode, split):
    from mscnn_b200 import capi, ops
    _, h, w, k, s, p = case
    rng = np.random.default_rng(13)
    x = _bf16_exact(rng.standard_normal((2, 64, h, w)).astype(np.float32))
    ref = pool(x, _pair(k), _pair(s), _pair(p), mode)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    out = ops.pool_forward(xp, k, s, capi.POOL_MAX if mode == "MAX" else capi.POOL_AVE, pad=p)
    got = ops.planes_to_nchw(out).cpu().numpy()
    assert got.shape == ref.shape
    if mode == "MAX":
        assert np.array_equal(got, ref)
    else:
        np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("mode", ["MAX", "AVE"])
@pytest.mark.parametrize("shape", [(2, 64, 7, 7), (8, 512, 24, 80), (3, 64, 1, 1), (2, 264, 9, 11), (2, 512, 5, 6), (1, 72, 33, 1)],
                         ids=["7x7", "24x80_c512", "1x1", "c264", "30px", "c72_33x1"])
def test_global_pooling(cuda, shape, mode, split):
    """kernel = the whole image: the CTA-wide reduction from 32 pixels up (7x7, 24x80), the per-output kernel below (1x1,
    5x6); C = 264 and 72 are padded planes of 320 and 128 channels, five and two blocks of eight 8-channel groups."""
    from mscnn_b200 import capi, ops
    n, c, h, w = shape
    rng = np.random.default_rng(14)
    x = _bf16_exact(rng.standard_normal(shape).astype(np.float32) + 0.25)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    out = ops.pool_forward(xp, None, 1, capi.POOL_MAX if mode == "MAX" else capi.POOL_AVE)
    assert out.shape == (n, 1, 1, (c + 63) // 64 * 64)
    got = ops.planes_to_nchw(out).cpu().numpy()
    if mode == "MAX":
        assert np.array_equal(got, x.max(axis=(2, 3), keepdims=True))
    else:
        ref = x.astype(np.float64).mean(axis=(2, 3), keepdims=True)
        np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)
        assert float(out.hi[..., c:].float().abs().max()) == 0.0 if c % 64 else True


def test_pool2d_dyn_n(cuda):
    from mscnn_b200 import capi, ops
    rng = np.random.default_rng(15)
    x = torch.from_numpy(rng.standard_normal((4, 64, 9, 12)).astype(np.float32)).to(cuda)
    xp = ops.nchw_to_planes(x, True)
    for kernel, stride, pad in [((3, 2), (2, 1), (1, 0)), (None, 1, 0)]:
        full = ops.pool_forward(xp, kernel, stride, capi.POOL_AVE, pad=pad)
        for count in (0, 1, 3, 6):
            out = ops.Planes(torch.full_like(full.hi, 7.0), torch.full_like(full.lo, 7.0), 64)
            dyn = torch.tensor([count], dtype=torch.int32, device=cuda)
            ops.pool_forward(xp, kernel, stride, capi.POOL_AVE, dyn=dyn, out=out, pad=pad)
            torch.cuda.synchronize()
            k = min(count, 4)
            assert torch.equal(out.hi[:k], full.hi[:k]) and torch.equal(out.lo[:k], full.lo[:k])
            assert bool((out.hi[k:] == 7.0).all()) and bool((out.lo[k:] == 7.0).all())


def test_general_entry_equals_the_square_entry_bitwise(cuda):
    from mscnn_b200 import capi, ops
    rng = np.random.default_rng(16)
    xp = ops.nchw_to_planes(torch.from_numpy(rng.standard_normal((2, 64, 9, 15)).astype(np.float32)).to(cuda), True)
    for mode in (capi.POOL_MAX, capi.POOL_AVE):
        for k, s in [(2, 2), (3, 2), (2, 1)]:
            a = ops.pool_forward(xp, k, s, mode)
            b = ops.pool_forward(xp, (k, k), (s, s), mode)
            assert torch.equal(a.hi, b.hi) and torch.equal(a.lo, b.lo)


# ---- one net with every new geometry, against the reference's own layers ----
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
def test_geometry_net_matches_the_reference_layers(side_stream, graph):
    """Blob by blob within the 1e-3 gate of the fp32-faithful mode, at two input sizes with a reshape_input in between:
    the 2x2 / 2 pool is computed in the strided convolution's epilogue at the first size and by itself at the second
    (odd extents), and the global pool follows the size."""
    from mscnn_b200 import net as mnet, synth
    mnet.set_precision("fp32")
    golden = np.load(GOLDEN)
    h0, w0 = GEOMETRY_SIZES[0]
    net = mnet.Net(geometry_net(h0, w0))
    net.set_params(synth.make_weights(net.layers()))
    net.set_graph(graph)
    replays = 0
    for h, w in GEOMETRY_SIZES + GEOMETRY_SIZES[:1]:
        net.reshape_input("data", 2, 3, h, w)
        for _ in range(3 if graph else 1):
            net.forward(data=synth.make_images(2, h, w))
            replays += int(net.graph_replayed())
        for name in GEOMETRY_BLOBS:
            if name == "c_rect" and (h, w) == GEOMETRY_SIZES[0]:
                continue      # pooled in its own epilogue and read by nothing else: the un-pooled blob is not written
            want = golden[f"{h}x{w}/{name}"]
            got = net.blob(name).reshape(want.shape)
            err = float(np.abs(got - want).max()) / float(np.sqrt((want.astype(np.float64) ** 2).mean()))
            assert err <= 1e-3, (h, w, name, err)
    assert replays >= (3 if graph else 0) and (graph or replays == 0)
