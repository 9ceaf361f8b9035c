"""The geometry of the Caltech and CityPersons nets, layer by layer, against plain references: ROIPooling and ROIAlign
with rectangular bins (the nets pool 8 rows x 4 columns), LFCN heads with 5x3 and 7x5 kernels, roi_c1 and fc6 on an
8x4 ROI grid, and BoxOutput with 1:2 pedestrian anchors (field_h = 2 field_w).

In each of these a swap of h and w still gives consistent shapes down the net, so only the values can tell.  The bars
are those of the square-geometry tests: ROIPooling bit-exact against oracle.port (test_detect_gpu.test_roi_pool_parity),
ROIAlign within one output rounding (test_roi_align_parity), convolutions against fp64 (test_conv_gpu), BoxOutput bit for
bit on scores and within 3e-7 on coordinates (test_detect_gpu._compare_boxes)."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import port
from test_conv_gpu import _ref_conv, _report
from test_detect_gpu import _compare_boxes, _maps, _run_cpu, _run_gpu
from test_device_rows_gpu import SENT_BF16, _bits, _box_n, _check_counts, _desc_like, _fill, _special_rois

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).resolve().parent / "golden"


def _bf16_exact(a):
    return torch.from_numpy(a).bfloat16().float().numpy()


def _same(got, ref, what, swapped=None):
    """Bit-exact, with the first differing (roi, channel, row, column) indices on failure, and how many elements
    differ when the bins are read as computed with pooled_h and pooled_w swapped (swapped(): that reference)."""
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bad = np.argwhere(got != ref)
    if len(bad):
        msg = [f"{what}: {len(bad)}/{got.size} elements differ; first at {bad[:6].tolist()}"]
        for i in bad[:4]:
            t = tuple(i)
            msg.append(f"  at {t}: got {got[t]:.6f} ref {ref[t]:.6f}")
        if swapped is not None:
            r, c, ph, pw = got.shape
            msg.append(f"  read as pooled_h={pw}, pooled_w={ph}: "
                       f"{int((got.reshape(r, c, pw, ph) != swapped()).sum())} elements differ")
        pytest.fail("\n".join(msg))


def _worst(got, ref, rms):
    """max |got - ref| / (|ref| + rms(ref)): the error in the units of the bars."""
    return float(((got.double() - ref).abs() / (ref.abs() + rms)).max())


def _ped_rois(rng, n, img_w, img_h, r, scale, bins):
    """test_roi_pool_parity's mix (random boxes, the dummy, a malformed, an outside and a half-pixel ROI), then a third
    tall, narrow pedestrian boxes (h = 2.4 w) and a sixth boxes smaller than one bin of the feature map."""
    rois = _special_rois(rng, n, img_w, img_h, r)
    k = r // 3
    bw = rng.uniform(6, 140, k)
    x1, y1 = rng.uniform(-10, img_w - 10, k), rng.uniform(-20, img_h - 40, k)
    rois[4:4 + k] = np.stack([rng.integers(0, n, k), x1, y1, x1 + bw, y1 + 2.4 * bw], axis=1)
    m = r // 6
    x1, y1 = rng.uniform(0, img_w, m), rng.uniform(0, img_h, m)
    bw, bh = rng.uniform(0, bins[1] / scale, m), rng.uniform(0, bins[0] / scale, m)
    rois[4 + k:4 + k + m] = np.stack([rng.integers(0, n, m), x1, y1, x1 + bw, y1 + bh], axis=1)
    return rois.astype(np.float32)


BINS = [(8, 4), (4, 8), (3, 5), (1, 7)]


# ------------------------------------------------------------------------------------------------------- ROIPooling
@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
# C = 512: every lane pools two channel groups (the DUAL path)
@pytest.mark.parametrize("c", [64, 128, 512])
@pytest.mark.parametrize("bins", BINS, ids=[f"{h}x{w}" for h, w in BINS])
def test_roi_pool_rect_parity(cuda, bins, c, split):
    from mscnn_b200 import ops
    ph, pw = bins
    rng = np.random.default_rng(1000 + 10 * ph + pw + c)
    n, h, w, r = 2, 24, 80, 240
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    for scale in (0.125, 0.25):
        rois = _ped_rois(rng, n, w / scale, h / scale, r, scale, bins)
        dr = torch.from_numpy(rois).to(cuda)
        for pad_ratio in (0.0, 0.25):
            ref = port.roi_pool(x, rois, ph, pw, scale, pad_ratio)
            out = ops.roi_pool_forward(xp, dr, r, bins, scale, pad_ratio)
            assert tuple(out.hi.shape) == (r, ph, pw, c)
            _same(ops.planes_to_nchw(out).cpu().numpy(), ref, f"roi_pool {bins} scale {scale} pad_ratio {pad_ratio}",
                  lambda: port.roi_pool(x, rois, pw, ph, scale, pad_ratio))


FUSED = [((8, 4), 64), ((8, 4), 512), ((3, 5), 128)]
ROI_CAP = 97


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("bins,c", FUSED, ids=[f"{b[0]}x{b[1]}-c{c}" for b, c in FUSED])
def test_roi_pool_rect_fused_and_device_rows(cuda, bins, c, split):
    """The nets' org || ctx pair as one launch (offsets 0 and C) == the Concat of two oracle ROIPoolings; then the
    device-row-count form: rows below the count equal the launch without one bit for bit, rows at or above it keep
    their sentinel (test_device_rows_gpu)."""
    from mscnn_b200 import ops
    ph, pw = bins
    rng = np.random.default_rng(77 + c + ph)
    n, h, w, scale = 2, 48, 96, 0.25
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    rois = _ped_rois(rng, n, w / scale, h / scale, ROI_CAP, scale, bins)
    ref = port.concat_channels(port.roi_pool(x, rois, ph, pw, scale, 0.0), port.roi_pool(x, rois, ph, pw, scale, 0.25))
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    dr = torch.from_numpy(rois).to(cuda)

    def planes():
        hi = torch.empty((ROI_CAP, ph, pw, 2 * c), dtype=torch.bfloat16, device=cuda)
        p = ops.Planes(hi, torch.empty_like(hi) if split else None, 2 * c)
        for t in [p.hi] + ([p.lo] if split else []):
            _fill(t)
        return p

    full = ops.roi_pool_multi_forward(xp, dr, ROI_CAP, bins, scale, (0.0, 0.25), (0, c), out=planes(), out_channels=2 * c)
    _same(ops.planes_to_nchw(full).cpu().numpy(), ref, f"fused roi_pool {bins}")
    full_t = [full.hi] + ([full.lo] if split else [])
    out = planes()
    outs = [out.hi] + ([out.lo] if split else [])
    _check_counts(cuda, lambda dyn: ops.roi_pool_multi_forward(xp, dr, ROI_CAP, bins, scale, (0.0, 0.25), (0, c),
                                                               out=out, out_channels=2 * c, dyn=dyn),
                  outs, full_t, 1, ROI_CAP, f"roi_pool {bins} C={c}", counts=[0, 1, ROI_CAP // 2, ROI_CAP - 3, ROI_CAP])
    assert int((_bits(out.hi) == SENT_BF16).sum()) == 0     # the last count wrote every row


# -------------------------------------------------------------------------------------------------------- ROIAlign
ALIGN_BINS = [(4, 7), (8, 4)]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("pad_ratio,scale", [(0.0, 0.125), (0.25, 0.25)])
@pytest.mark.parametrize("bins", ALIGN_BINS, ids=[f"{h}x{w}" for h, w in ALIGN_BINS])
def test_roi_align_rect_parity(cuda, bins, pad_ratio, scale, split):
    """At test_roi_align_parity's bars: fp32 interpolation in the reference's order, stored as bf16 planes."""
    from mscnn_b200 import ops
    ph, pw = bins
    rng = np.random.default_rng(23 + ph * pw)
    n, c, h, w, r = 2, 128, 24, 40, 150
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    rois = _ped_rois(rng, n, w / scale, h / scale, r, scale, bins)
    rois[4 + r // 3 + r // 6] = [0, 0, 0, w / scale - 1, h / scale - 1]
    ref = port.roi_align(x, rois, ph, pw, scale, pad_ratio)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    out = ops.roi_align_forward(xp, torch.from_numpy(rois).to(cuda), r, bins, scale, pad_ratio)
    got = ops.planes_to_nchw(out).cpu().numpy()
    assert got.shape == ref.shape == (r, c, ph + 1, pw + 1)
    assert not got[1].any() and not got[2].any()
    np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)
    assert np.array_equal(got == 0, ref == 0)


# ------------------------------------------------------------------------------------------------ rectangular heads
HEAD_K = [((5, 3), (2, 1)), ((7, 5), (3, 2))]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("cin", [64, 512])
@pytest.mark.parametrize("cout", [6, 9])
@pytest.mark.parametrize("k,pad", HEAD_K, ids=["5x3", "7x5"])
def test_conv_head_rect(cuda, k, pad, cout, cin, split):
    """The pedestrian LFCN heads (kernel_h x kernel_w 5x3 and 7x5, "same" padding): the head-taps path takes square
    kernels only, so these run the direct implicit GEMM with fp32 NCHW output.  At test_conv_head_f32_nchw's bars, on a
    single pixel, a width below kernel_w, 12x40 and a width past one 128-pixel tile."""
    from mscnn_b200 import ops
    kh, kw = k
    g = torch.Generator(device="cpu").manual_seed(10 * kh + kw + cout + cin)
    for n, h, w in [(1, 1, 1), (2, 6, kw - 1), (3, 12, 40), (1, 5, 129)]:
        x = torch.randn((n, cin, h, w), generator=g).to(cuda)
        wt = (torch.randn((cout, cin, kh, kw), generator=g) * 0.02).to(cuda)
        b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
        got = ops.conv_forward(ops.nchw_to_planes(x, split), ops.pack_conv_weights(wt, b, split), pad, relu=False,
                               out_f32=True)
        torch.cuda.synchronize()
        if split:
            ref = _ref_conv(x, wt, b, pad, False)
        else:
            ref = _ref_conv(x.bfloat16().float(), wt.bfloat16().float(), b, pad, False)
        assert got.shape == ref.shape == (n, cout, h, w)
        rms = float(ref.pow(2).mean().sqrt())
        # the direct path sums K = 3 * Cin * kh * kw split products in one fp32 accumulator whose adds truncate:
        # at Cin 512, 7x5 (K = 53,760) that reaches 2.8e-4 rms(ref) (measured on an H100), so the bar is the one
        # test_net_gpu.test_head_taps_path_equals_direct_conv sets for this path, 5e-4 rms(ref)
        _report(f"head {kh}x{kw} shape={(n, h, w)}", got, ref, 1e-4, (5e-4 if split and cin == 512 else 1e-4) * rms)
        print(f"head {kh}x{kw} Cin {cin} shape={(n, h, w)}: {_worst(got, ref, rms):.2e}")


# ------------------------------------------------------------------------------------- roi_c1 and fc6 on 8x4 grids
@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("r", [1, 3, 4, 5, 127, 128, 129, 2001])
def test_roi_c1_fc6_on_8x4_grid(cuda, r, split):
    """roi_c1 (3x3 pad 1, 1024 -> 512, ReLU) on [R, 1024, 8, 4]: one pixel box spans several ROIs, so every tile has
    halos at the edges of several images.  Then fc6 (K = 8 * 4 * 512 = 16384 -> 2048, ReLU) and cls_pred 2 / bbox_pred 8
    with fp32 output, each against fp64 of its own input.  roi_c1 also runs with a device row count of R - 3."""
    from mscnn_b200 import capi, ops
    g = torch.Generator(device="cpu").manual_seed(8004 + r)
    cin, cout, ph, pw = 1024, 512, 8, 4
    x = torch.randn((r, cin, ph, pw), generator=g).to(cuda)
    wt = (torch.randn((cout, cin, 3, 3), generator=g) * (2.0 / (cin * 9)) ** 0.5).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    wp = ops.pack_conv_weights(wt, b, split)
    y = ops.conv_forward(xp, wp, 1, relu=True)
    got = ops.planes_to_nchw(y)
    torch.cuda.synchronize()
    # the bars of test_conv_planes, except the absolute term in bf16: fp32 accumulation over K = 9216 (twice the K of
    # test_conv_device_rows's roi_c1, whose 3e-5 rms(ref) it exceeds at R = 2001) takes the split path's 1e-4 rms(ref)
    if split:
        ref = _ref_conv(x, wt, b, 1, True)
        rms = float(ref.pow(2).mean().sqrt())
        _report(f"roi_c1 R={r}", got, ref, 1e-4, 1e-4 * rms)
    else:
        ref = _ref_conv(x.bfloat16().float(), wt.bfloat16().float(), b, 1, True)
        rms = float(ref.pow(2).mean().sqrt())
        _report(f"roi_c1 R={r}", got, ref, 2.0 ** -8, 1e-4 * rms)
    kind = "split" if split else "bf16"
    print(f"roi_c1 R={r} {kind}: {_worst(got, ref, rms):.2e}")
    del ref

    # the device row count: rows below R - 3 bit for bit, rows from the count rounded up to the pixel box untouched
    full_t = [y.hi] + ([y.lo] if split else [])
    out = ops.Planes(torch.empty_like(y.hi), None if y.lo is None else torch.empty_like(y.lo), y.channels)
    outs = [out.hi] + ([out.lo] if split else [])
    box_n = _box_n(_desc_like(xp, wp, 1, capi.OUT_NHWC_BF16))
    _check_counts(cuda, lambda dyn: ops.conv_forward(xp, wp, 1, relu=True, dyn=dyn, out=out), outs, full_t, box_n, r,
                  f"roi_c1 R={r} box_n={box_n}", counts=[r - 3])

    # fc6 over the NHWC flattening of the 8x4x512 grid, weights in Caffe's NCHW flattening
    kin = cout * ph * pw
    w6 = (torch.randn((2048, kin), generator=g) * (2.0 / kin) ** 0.5).to(cuda)
    b6 = (torch.randn((2048,), generator=g) * 0.1).to(cuda)
    flat = ops.Planes(y.hi.view(r, 1, 1, -1), None if y.lo is None else y.lo.view(r, 1, 1, -1), kin)
    f6 = ops.conv_forward(flat, ops.pack_fc_weights(w6, b6, split, cout, ph, pw), 0, relu=True)
    got6 = ops.planes_to_nchw(f6).view(r, 2048)
    xin, win = got.double().reshape(r, -1), (w6 if split else w6.bfloat16().float()).double()
    ref6 = torch.relu(xin @ win.t() + b6.double())
    rms6 = float(ref6.pow(2).mean().sqrt())
    # K = 16384 (ten times test_inner_product's fc6): the truncating fp32 accumulation reaches 1.2e-4 relative in
    # the split path and 2.7e-5 rms(ref) in bf16 (measured on an H100), so fc6 takes test_inner_product's bar for the
    # fc that follows fc6 (2e-4) in the split path, and the split path's absolute term in bf16
    if split:
        _report(f"fc6 R={r}", got6, ref6, 2e-4, 2e-4 * rms6)
    else:
        _report(f"fc6 R={r}", got6, ref6, 2.0 ** -8, 1e-4 * rms6)
    print(f"fc6 R={r} {kind}: {_worst(got6, ref6, rms6):.2e}")
    for name, nout in (("cls_pred", 2), ("bbox_pred", 8)):
        w2 = (torch.randn((nout, 2048), generator=g) * 0.05).to(cuda)
        b2 = (torch.randn((nout,), generator=g) * 0.1).to(cuda)
        got2 = ops.conv_forward(f6, ops.pack_fc_weights(w2, b2, split, 2048, 1, 1), 0, relu=False, out_f32=True).view(r, nout)
        torch.cuda.synchronize()
        if split:
            ref2 = ref6 @ w2.double().t() + b2.double()
            _report(f"{name} R={r}", got2, ref2, 2e-4, 2e-4 * float(ref2.pow(2).mean().sqrt()))
        else:
            ref2 = got6.double() @ w2.bfloat16().double().t() + b2.double()
            _report(f"{name} R={r}", got2, ref2, 1e-5, 1e-5 * float(ref2.pow(2).mean().sqrt()))


# ------------------------------------------------------------------------------------- BoxOutput, pedestrian anchors
CALTECH_BOX = dict(field_w=[30, 42, 60, 84, 120, 168, 240], field_h=[60, 84, 120, 168, 240, 336, 480],
                   rate=[8, 8, 16, 16, 32, 32, 64], fg_thr=-5.0, iou_thr=0.65, field_whr=2.0, field_xyr=2.0,
                   max_nms_num=2000)
CITYPERSONS_BOX = dict(field_w=[30, 42, 60, 84, 120, 168, 240, 336], field_h=[60, 84, 120, 168, 240, 336, 480, 672],
                       rate=[8, 8, 16, 16, 32, 32, 64, 64], fg_thr=-3.0, iou_thr=0.65, field_whr=2.0, field_xyr=2.0,
                       max_nms_num=2000, bbox_mean=[0, 0, 0, 0], bbox_std=[0.1, 0.1, 0.2, 0.2])
BOX_NETS = {"caltech": (CALTECH_BOX, "e2e_caltech_7s_240x320.npz"),
            "citypersons": (CITYPERSONS_BOX, "e2e_citypersons_cascade_192x384.npz")}


@pytest.mark.parametrize("net", list(BOX_NETS))
def test_box_output_pedestrian_anchors(cuda, net):
    """The shipped box_output_param of the Caltech (no bbox normalisation) and CityPersons (normalised) nets, batch 2,
    on seeded maps of the fixture's LFCN shapes and on the fixture's own LFCN maps.  The oracle's answer with field_w
    and field_h swapped differs, so the case tells the two apart."""
    kw, fixture = BOX_NETS[net]
    g = np.load(GOLD / fixture)
    heads = sorted(k for k in g.files if k.startswith("LFCN_"))       # the BoxOutput's bottom order
    assert len(heads) == len(kw["rate"])
    real = [np.ascontiguousarray(g[k]) for k in heads]
    rng = np.random.default_rng(len(heads))
    seeded = _maps(rng, 2, 6, [m.shape[2:] for m in real], box_scale=1.0, bg_bias=1.0)
    for what, maps in (("seeded", seeded), ("fixture", real)):
        c = _run_cpu(maps, **kw)
        frac = _compare_boxes(_run_gpu(cuda, maps, **kw), c)
        assert c[3] > 50, (what, c[3])
        print(f"[{net} {what}] {c[3]} proposals, {list(c[2])} per image, coordinates bit-identical {frac:.4f}")
        sw = _run_cpu(maps, **dict(kw, field_w=kw["field_h"], field_h=kw["field_w"]))
        assert sw[0].shape != c[0].shape or not np.array_equal(sw[0], c[0]), (what, "field_w / field_h swap unseen")
