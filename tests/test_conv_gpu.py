"""Parity of the wgmma implicit-GEMM convolution (mscnn_conv_forward) against an fp64
convolution of the same operands.

Reference semantics: ConvolutionLayer::Forward_cpu = im2col + sgemm + bias
(/root/reference/src/caffe/layers/conv_layer.cpp:25-40, base_conv_layer.cpp:257-280) and the
reference's own test tolerance for it, 1e-4 absolute on O(1) data
(src/caffe/test/test_convolution_layer.cpp:231-265).  Tolerances used here:
  split-bf16 ("fp32-faithful") path: |err| <= 1e-4 * (|ref| + rms(ref)).  The 3-term split has a
  per-product relative error of ~2^-16; over K random-sign terms that is ~1e-5 rms(ref) typical,
  ~5e-5 rms(ref) at the 4.5-sigma tail of a 32k-element tensor.
  plain bf16 path: exact products of bf16-rounded operands, so vs fp64 conv of the ROUNDED
  operands |err| <= 1e-5 scale for fp32 output, one bf16 ulp (2^-8 rel) for bf16 planes.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ref_conv(x, w, b, pad, relu):
    y = F.conv2d(x.double(), w.double(), None if b is None else b.double(), padding=pad)
    return torch.relu(y) if relu else y


def _report(name, got, ref, tol_rel, tol_abs):
    err = (got.double() - ref).abs()
    lim = tol_rel * ref.abs() + tol_abs
    bad = err > lim
    if bad.any():
        idx = bad.nonzero()
        msg = [f"{name}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; "
               f"max err {float(err.max()):.3e}, ref rms {float(ref.pow(2).mean().sqrt()):.3e}"]
        for d in range(idx.shape[1]):
            u = idx[:, d].unique()
            msg.append(f"  dim{d}: {u.numel()} distinct bad indices, first {u[:16].tolist()}")
        for i in idx[:8]:
            t = tuple(i.tolist())
            msg.append(f"  at {t}: got {float(got[t]):.6f} ref {float(ref[t]):.6f}")
        pytest.fail("\n".join(msg))


# Case names are test ids and stay stable.  Some name the operand-delivery variant a shape once selected (mt_*: several
# M sub-tiles per CTA tile; rowshare_*: a shared haloed activation row; ring256_*: separate activation and weight
# rings); the comments say what each shape exercises in the current kernel.
CASES = [
    # name,            N, Cin, H,  W, Cout, k, pad
    ("trunk64",        1, 64, 16, 32, 64, 3, 1),
    ("trunk128",       2, 64, 12, 40, 128, 3, 1),
    ("trunk256",       1, 128, 24, 20, 256, 3, 1),
    ("trunk512_2nt",   1, 128, 8, 16, 512, 3, 1),
    ("ragged",         3, 64, 9, 30, 64, 3, 1),
    ("roi_c1_like",    7, 128, 7, 7, 128, 3, 0),
    ("conv1x1",        1, 64, 8, 24, 64, 1, 0),
    ("deepK",          1, 512, 6, 40, 128, 3, 1),
    # 3 input channels padded to one 64-channel chunk: conv1_1-like layers with Cout != 64
    ("c3_n48",         2, 3, 21, 150, 48, 3, 1),
    ("c3_n128",        1, 3, 20, 36, 128, 3, 1),
    # many more M tiles than SMs: every persistent CTA walks several tiles through the ring
    ("mt_n64",         2, 64, 128, 160, 64, 3, 1),
    ("mt_n128",        2, 64, 128, 320, 128, 3, 1),
    # W a multiple of 128 with narrow N: 128x1 boxes, fat stages, one and two channel chunks, more tiles than ring slots
    ("rowshare_n64",   1, 64, 6, 256, 64, 3, 1),
    ("rowshare_n128",  2, 128, 5, 384, 128, 3, 1),
    ("rowshare_many",  2, 64, 40, 512, 64, 3, 1),
    # BLOCK_N = 256 on 128x1 boxes: term-major k-blocks with single operand tiles per stage -- the variant conv3_x
    # takes at 768x2560.  Even / odd M-tile counts, one and two n tiles, 4 and 8 channel chunks, more tiles than SMs.
    ("ring256_halo",   1, 256, 6, 256, 256, 3, 1),
    ("ring256_odd",    1, 256, 5, 384, 256, 3, 1),
    ("ring256_2nt",    2, 256, 5, 640, 512, 3, 1),
    ("ring256_c512",   1, 512, 3, 384, 512, 3, 1),
    ("ring256_many",   2, 256, 40, 640, 256, 3, 1),
    # BLOCK_N = 256 on 2-D boxes: conv4_x / conv5_x geometry, odd tile count
    ("ring256_box2d",  1, 256, 24, 40, 512, 3, 1),
    ("ring256_box2d_odd", 3, 256, 12, 40, 256, 3, 1),
]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_planes(cuda, case, split):
    from mscnn_b200 import ops
    name, n, cin, h, w, cout, k, pad = case
    g = torch.Generator(device="cpu").manual_seed(1706)
    x = torch.randn((n, cin, h, w), generator=g).to(cuda)
    wt = (torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    wp = ops.pack_conv_weights(wt, b, split)
    yp = ops.conv_forward(xp, wp, pad, relu=True)
    torch.cuda.synchronize()
    got = ops.planes_to_nchw(yp)
    torch.cuda.synchronize()
    if split:
        ref = _ref_conv(x, wt, b, pad, True)
        rms = float(ref.pow(2).mean().sqrt())
        _report(name, got, ref, 1e-4, 1e-4 * rms)
    else:
        ref = _ref_conv(x.bfloat16().float(), wt.bfloat16().float(), b, pad, True)
        rms = float(ref.pow(2).mean().sqrt())
        _report(name, got, ref, 2.0 ** -8, 1e-5 * rms)


VARIANT_CASES = [c for c in CASES if c[0].startswith("ring256") or c[0] in ("trunk256", "trunk512_2nt", "rowshare_n128")]


@pytest.mark.parametrize("case", VARIANT_CASES, ids=[c[0] for c in VARIANT_CASES])
def test_conv_variants_bit_identical(cuda, case, monkeypatch):
    """Operand-delivery variants of one layer.  The default plan is repeatable bit for bit; MSCNN_NO_FAT (term-major
    k-blocks: all of hi*hi, then hi*lo, then lo*hi) is the plan BLOCK_N = 256 layers always take, so it is bit-identical
    there, and another summation order elsewhere, held to fp64 only.  Every variant must be within 1e-4 of the fp64
    convolution."""
    from mscnn_b200 import ops
    name, n, cin, h, w, cout, k, pad = case
    g = torch.Generator(device="cpu").manual_seed(1707)
    x = torch.randn((n, cin, h, w), generator=g).to(cuda)
    wt = (torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, True)
    wp = ops.pack_conv_weights(wt, b, True)
    ref = _ref_conv(x, wt, b, pad, True)
    rms = float(ref.pow(2).mean().sqrt())

    def run(**env):
        for kk, v in env.items():
            monkeypatch.setenv(kk, v)
        ops.reload_config()
        try:
            y = ops.conv_forward(xp, wp, pad, relu=True)
            got = ops.planes_to_nchw(y)
            torch.cuda.synchronize()
            _report(f"{name} {env}", got, ref, 1e-4, 1e-4 * rms)
            return y.hi.clone(), y.lo.clone()
        finally:
            for kk in env:
                monkeypatch.delenv(kk)
            ops.reload_config()

    def same_as(base, other, what):
        if not (torch.equal(base[0], other[0]) and torch.equal(base[1], other[1])):
            d = (base[0] != other[0]) | (base[1] != other[1])
            pytest.fail(f"{name}: {what} differs from the default build in {int(d.sum())}/{d.numel()} elements, "
                        f"first at {d.nonzero()[:4].tolist()}")

    base = run()
    same_as(base, run(), "a second run")
    nofat = run(MSCNN_NO_FAT="1")
    cpad = (cout + 63) // 64 * 64
    if cpad % 256 == 0:
        same_as(base, nofat, "MSCNN_NO_FAT")


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("k,pad", [(5, 2), (7, 3), (1, 0)])
def test_conv_head_f32_nchw(cuda, k, pad, split):
    """Narrow proposal heads: Cout = 9 (LFCN_*), fp32 NCHW output."""
    from mscnn_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(7)
    n, cin, h, w, cout = 2, 128, 12, 40, 9
    x = torch.randn((n, cin, h, w), generator=g).to(cuda)
    wt = (torch.randn((cout, cin, k, k), generator=g) * 0.02).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    wp = ops.pack_conv_weights(wt, b, split)
    got = ops.conv_forward(xp, wp, pad, relu=False, out_f32=True)
    torch.cuda.synchronize()
    if split:
        ref = _ref_conv(x, wt, b, pad, False)
        _report("head", got, ref, 1e-4, 1e-4 * float(ref.pow(2).mean().sqrt()))
    else:
        ref = _ref_conv(x.bfloat16().float(), wt.bfloat16().float(), b, pad, False)
        _report("head", got, ref, 1e-4, 1e-4 * float(ref.pow(2).mean().sqrt()))  # fp32 accumulation over K=6272


def _head_taps(x, wt, b, split):
    """The Net's k x k head path: the horizontal taps as GEMM columns (mscnn_pack_head_weights, a k x 1 convolution
    into pixel-major fp32 rows P[pixel][dx * Cout + co]), then mscnn_head_gather sums P over dx and adds the bias."""
    from mscnn_b200 import capi, ops
    cout, cin, k, _ = wt.shape
    n, _, h, w = x.shape
    n_pad = (k * cout + 63) // 64 * 64
    cin_pad = ops.pad64(cin)
    hi = torch.empty((n_pad, k, 1, cin_pad), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi) if split else None
    L = capi.lib()
    stream = torch.cuda.current_stream().cuda_stream
    capi.check(L.mscnn_pack_head_weights(capi.ptr(wt), capi.ptr(hi), capi.ptr(lo), cout, cin, k, n_pad, cin_pad,
                                         stream), "pack_head_weights")
    wp = ops.PackedWeights(hi, lo, torch.zeros(n_pad, dtype=torch.float32, device=x.device), n_pad, k, 1)
    p = ops.conv_forward(ops.nchw_to_planes(x, split), wp, (k // 2, 0), relu=False, out_mode=capi.OUT_NHWC_F32)
    assert tuple(p.shape) == (n, h, w, n_pad)
    y = torch.empty((n, cout, h, w), dtype=torch.float32, device=x.device)
    capi.check(L.mscnn_head_gather(capi.ptr(p), n_pad, capi.ptr(b), capi.ptr(y), n, h, w, cout, k, k // 2, stream),
               "head_gather")
    return y


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("cin", [64, 512])
@pytest.mark.parametrize("cout", [6, 9])
@pytest.mark.parametrize("k", [3, 5, 7])
def test_conv_head_taps(cuda, k, cout, cin, split):
    """The LFCN heads as the Net runs them (the only non-square convolution and the only OUT_NHWC_F32 user), vs fp64,
    at test_conv_head_f32_nchw's bars.  Widths and heights below the reach of the taps, a single pixel, and a width
    past one 128-pixel tile."""
    g = torch.Generator(device="cpu").manual_seed(100 * k + cout + cin)
    for n, h, w in [(1, 1, 1), (2, 3, k - 1), (3, 12, 40), (1, 5, 129)]:
        x = torch.randn((n, cin, h, w), generator=g).to(cuda)
        wt = (torch.randn((cout, cin, k, k), generator=g) * 0.02).to(cuda)
        b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
        got = _head_taps(x, wt, b, split)
        torch.cuda.synchronize()
        if split:
            ref = _ref_conv(x, wt, b, k // 2, False)
        else:
            ref = _ref_conv(x.bfloat16().float(), wt.bfloat16().float(), b, k // 2, False)
        _report(f"head taps k={k} shape={(n, h, w)}", got, ref, 1e-4, 1e-4 * float(ref.pow(2).mean().sqrt()))


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_inner_product(cuda, split):
    """InnerProduct (inner_product_layer.cpp:84-97): Y = X W^T + b with X the NCHW flattening of
    a [R,C,H,W] bottom; weights are re-ordered to the NHWC flattening at pack time."""
    from mscnn_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(11)
    r, c, h, w, nout = 300, 64, 5, 5, 128
    x = torch.randn((r, c, h, w), generator=g).to(cuda)
    wt = (torch.randn((nout, c * h * w), generator=g) * 0.02).to(cuda)
    b = (torch.randn((nout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    flat = ops.Planes(xp.hi.view(r, 1, 1, -1), None if xp.lo is None else xp.lo.view(r, 1, 1, -1),
                      h * w * 64)
    wp = ops.pack_fc_weights(wt, b, split, c, h, w)
    yp = ops.conv_forward(flat, wp, 0, relu=True)
    got = ops.planes_to_nchw(yp).view(r, nout)
    # second, narrow fc with fp32 output (cls_pred / bbox_pred shape class)
    wt2 = (torch.randn((25, nout), generator=g) * 0.05).to(cuda)
    b2 = (torch.randn((25,), generator=g) * 0.1).to(cuda)
    wp2 = ops.pack_fc_weights(wt2, b2, split, nout, 1, 1)
    got2 = ops.conv_forward(yp, wp2, 0, relu=False, out_f32=True).view(r, 25)
    torch.cuda.synchronize()
    xin, win = (x, wt) if split else (x.bfloat16().float(), wt.bfloat16().float())
    ref = torch.relu(xin.view(r, -1).double() @ win.double().t() + b.double())
    rms = float(ref.pow(2).mean().sqrt())
    if split:
        _report("fc6", got, ref, 1e-4, 1e-4 * rms)
        ref2 = ref @ wt2.double().t() + b2.double()
        _report("fc_narrow", got2, ref2, 2e-4, 2e-4 * float(ref2.pow(2).mean().sqrt()))
    else:
        _report("fc6", got, ref, 2.0 ** -8, 1e-5 * rms)
        ref2 = got.double() @ wt2.bfloat16().double().t() + b2.double()
        _report("fc_narrow", got2, ref2, 1e-5, 1e-5 * float(ref2.pow(2).mean().sqrt()))


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("shape", [(2, 21, 150), (1, 5, 40), (3, 40, 384), (1, 3, 129), (2, 160, 640)])
def test_conv1_1_tensor_core(cuda, split, shape):
    """conv1_1 as the single tensor-core kernel (descriptor-shifted pixel rows; the path the Net uses).
    Widths below / across / at multiples of the 128-pixel tile, more tiles than SMs in the last case."""
    from mscnn_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(4)
    n, h, w = shape
    x = (torch.randint(0, 256, (n, 3, h, w), generator=g).float()
         - torch.tensor([104.0, 117.0, 123.0]).view(1, 3, 1, 1)).to(cuda).contiguous()
    x[0, :, h // 2, w // 3] += 0.37          # not bf16-representable: exercises the lo plane of the input
    wt = (torch.randn((64, 3, 3, 3), generator=g) * (2.0 / 27) ** 0.5 / 64).to(cuda)
    b = (torch.randn((64,), generator=g) * 0.1).to(cuda)
    for relu in (True, False):
        yp = ops.conv1_tc_forward(x, wt, b, relu=relu, split=split)
        got = ops.planes_to_nchw(yp)
        torch.cuda.synchronize()
        if split:
            ref = _ref_conv(x, wt, b, 1, relu)
            rms = float(ref.pow(2).mean().sqrt())
            _report("conv1_1_tc", got, ref, 2e-5, 2e-5 * rms)
        else:
            ref = _ref_conv(x.bfloat16().float(), wt.bfloat16().float(), b, 1, relu)
            rms = float(ref.pow(2).mean().sqrt())
            _report("conv1_1_tc", got, ref, 2.0 ** -8, 1e-5 * rms)


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("shape", [(2, 64, 64, 192, 64), (1, 64, 128, 320, 128), (2, 128, 24, 80, 256), (3, 64, 10, 12, 64),
                                   # W % 128 == 0, narrow N: row-pair tiles with the pooling done in registers
                                   (1, 64, 8, 256, 64), (2, 128, 6, 128, 128), (2, 64, 64, 512, 64), (1, 64, 32, 384, 128)])
def test_conv_fused_pool(cuda, split, shape):
    """mscnn_conv_forward with pool_hi set == conv followed by mscnn_pool_forward, bit for bit; the
    pool-only form (no un-pooled store) gives the same pooled planes."""
    from mscnn_b200 import ops
    n, cin, h, w, cout = shape
    g = torch.Generator(device="cpu").manual_seed(21)
    x = torch.randn((n, cin, h, w), generator=g).to(cuda)
    wt = (torch.randn((cout, cin, 3, 3), generator=g) * (2.0 / (cin * 9)) ** 0.5).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    wp = ops.pack_conv_weights(wt, b, split)
    y_ref = ops.conv_forward(xp, wp, 1, relu=True)
    p_ref = ops.pool_forward(y_ref, 2, 2)
    y_both, p_both = ops.conv_forward(xp, wp, 1, relu=True, pool="both")
    p_only = ops.conv_forward(xp, wp, 1, relu=True, pool="only")
    torch.cuda.synchronize()
    assert torch.equal(y_both.hi, y_ref.hi)
    for cand in (p_both, p_only):
        assert torch.equal(cand.hi, p_ref.hi)
        if split:
            assert torch.equal(cand.lo, p_ref.lo)


def test_layout_roundtrip(cuda):
    from mscnn_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn((2, 70, 5, 37), generator=g).to(cuda)
    p = ops.nchw_to_planes(x, True)
    y = ops.planes_to_nchw(p)
    torch.cuda.synchronize()
    assert float((y - x).abs().max()) <= 2.0 ** -16 * float(x.abs().max())
    assert float(p.hi[..., 70:].float().abs().max()) == 0.0
    p1 = ops.nchw_to_planes(x, False)
    assert torch.equal(p1.hi[..., :70], x.permute(0, 2, 3, 1).bfloat16())
