"""Data-dependent row counts read on the device (mscnn_conv_desc.dyn_n, mscnn_pool_forward_dyn,
mscnn_roi_pool_multi_forward_dyn, mscnn_roi_align_forward_dyn).  Every layer behind BoxOutput runs this way: the launch
is sized for the cap and the kernel reads R from device memory.

Each case first holds a launch without a count to the reference (fp64 for the convolutions, the oracle port for the
pooling kernels).  Then it launches into outputs pre-filled with a NaN sentinel, with one device count whose value
changes between launches through the same pointer, as a graph replay changes it.  Rows below min(max(count, 0), cap)
must equal the launch without a count bit for bit.  Rows from the count rounded up to the kernel's row granularity
(the convolution's pixel box, one row elsewhere) must still hold the sentinel: the tiles were trimmed, not computed and
dropped."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

from oracle import port
from test_conv_gpu import _ref_conv, _report

pytestmark = pytest.mark.gpu

SENT_BF16 = 0x7FBF          # a quiet NaN no kernel produces
SENT_F32 = 0x7FC00001


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _sentinel(t):
    return SENT_BF16 if t.dtype == torch.bfloat16 else SENT_F32


def _fill(t):
    _bits(t).fill_(_sentinel(t))


def _counts(b, cap):
    return [-5, 0, 1, b - 1, b, b + 1, 2 * b + 7, cap - 1, cap, cap + 17]


def _check_counts(cuda, launch, outs, full, b, cap, what, counts=None):
    """launch(dyn) writes into `outs` (row dimension first); `full` are the same tensors of a launch without a count.
    counts: the device counts to try (default _counts(b, cap))."""
    dyn = torch.zeros(1, dtype=torch.int32, device=cuda)
    for count in _counts(b, cap) if counts is None else counts:
        for t in outs:
            _fill(t)
        dyn.fill_(count)
        launch(dyn)
        torch.cuda.synchronize()
        n = min(max(count, 0), cap)
        trimmed = min(-(-n // b) * b, cap)
        for k, (t, f) in enumerate(zip(outs, full)):
            got, want = _bits(t), _bits(f)
            if not torch.equal(got[:n], want[:n]):
                d = (got[:n] != want[:n]).nonzero()
                pytest.fail(f"{what} count={count} output {k}: {d.shape[0]} elements below the count differ from the "
                            f"launch without a count, first at {d[:4].tolist()}")
            tail = got[trimmed:]
            if not bool((tail == _sentinel(t)).all()):
                rows = (tail != _sentinel(t)).reshape(tail.shape[0], -1).any(1).nonzero().flatten() + trimmed
                pytest.fail(f"{what} count={count} (granularity {b}) output {k}: rows {rows[:8].tolist()} at or above "
                            f"{trimmed} were written")
            mid, mid_ref = got[n:trimmed], want[n:trimmed]
            assert bool(((mid == mid_ref) | (mid == _sentinel(t))).all()), (what, count, k)


# ------------------------------------------------------------------------------------------------ convolution
def _box_n(desc) -> int:
    from mscnn_b200 import capi
    buf = C.create_string_buffer(512)
    capi.check(capi.lib().mscnn_conv_plan_describe(C.byref(desc), buf, 512), "conv_plan_describe")
    m = re.search(r"box=(\d+)x(\d+)x(\d+)", buf.value.decode())
    assert m, buf.value
    return int(m.group(3))


def _desc_like(x, w, pad, out_mode):
    """The descriptor ops.conv_forward builds, for the plan query (pointers are only tested for NULL)."""
    from mscnn_b200 import capi
    fake = 0x10000
    n, h, wd, c = x.hi.shape
    d = capi.ConvDesc()
    d.x_hi, d.x_lo = fake, (fake if x.lo is not None else None)
    d.N, d.H, d.W, d.C = n, h, wd, c
    d.w_hi, d.w_lo, d.bias = fake, (fake if w.lo is not None else None), fake
    d.Cout, d.Cout_pad, d.KH, d.KW, d.pad_h, d.pad_w = w.cout, w.hi.shape[0], w.kh, w.kw, pad, pad
    d.relu, d.out_mode, d.dyn_n = 1, out_mode, fake
    if out_mode == capi.OUT_NHWC_BF16:
        d.y_hi, d.y_lo = fake, (fake if x.lo is not None else None)
    else:
        d.y_f32 = fake
    return d


CAP = 300
CONV_CASES = [
    # name,         Cin, H, W, Cout, k, pad, kind
    ("roi_c1",      512, 7, 7, 512, 3, 0, "conv"),      # <256, false>, 5x5 output
    ("roi_c1_wider", 512, 5, 5, 512, 3, 1, "conv"),
    ("fc6",          64, 7, 7, 512, 0, 0, "fc"),        # 1x1 over the 7*7*64 NHWC flattening
    ("cls_pred",    512, 1, 1, 5, 0, 0, "fc_f32"),      # NCHW fp32, BLOCK_N 32
    ("bbox_pred",   512, 1, 1, 20, 0, 0, "fc_f32"),
]


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_device_rows(cuda, case, split):
    from mscnn_b200 import capi, ops
    name, cin, h, w, cout, k, pad, kind = case
    g = torch.Generator(device="cpu").manual_seed(300 + len(name))
    x = torch.randn((CAP, cin, h, w), generator=g).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    xin = x if split else x.bfloat16().float()
    if kind == "conv":
        wt = (torch.randn((cout, cin, k, k), generator=g) * (2.0 / (cin * k * k)) ** 0.5).to(cuda)
        wp = ops.pack_conv_weights(wt, b, split)
        win = wt if split else wt.bfloat16().float()
        ref = _ref_conv(xin, win, b, pad, True)
    else:
        kin = cin * h * w
        wt = (torch.randn((cout, kin), generator=g) * (2.0 / kin) ** 0.5).to(cuda)
        wp = ops.pack_fc_weights(wt, b, split, cin, h, w)
        xp = ops.Planes(xp.hi.view(CAP, 1, 1, -1), None if xp.lo is None else xp.lo.view(CAP, 1, 1, -1), h * w * xp.hi.shape[3])
        win = wt if split else wt.bfloat16().float()
        ref = xin.reshape(CAP, -1).double() @ win.double().t() + b.double()
        if kind == "fc":
            ref = torch.relu(ref)
        ref = ref.view(CAP, cout, 1, 1)
    relu = kind != "fc_f32"
    f32 = kind == "fc_f32"
    out_mode = capi.OUT_NCHW_F32 if f32 else capi.OUT_NHWC_BF16

    full = ops.conv_forward(xp, wp, pad, relu=relu, out_f32=f32)
    torch.cuda.synchronize()
    rms = float(ref.pow(2).mean().sqrt())
    if f32:
        _report(name, full, ref, 1e-4, 1e-4 * rms)
        full_t = [full]
    else:
        got = ops.planes_to_nchw(full)
        torch.cuda.synchronize()
        if split:
            _report(name, got, ref, 1e-4, 1e-4 * rms)
        else:
            # one bf16 rounding of the output, plus the tensor core's fp32 accumulation over K = 4608 (roi_c1), which
            # reaches 1.5e-5 rms(ref) on a handful of the 3.8M outputs (measured on an H100)
            _report(name, got, ref, 2.0 ** -8, 3e-5 * rms)
        full_t = [full.hi] + ([full.lo] if full.lo is not None else [])

    box_n = _box_n(_desc_like(xp, wp, pad, out_mode))
    if f32:
        out = torch.empty_like(full)
        outs = [out]
    else:
        out = ops.Planes(torch.empty_like(full.hi), None if full.lo is None else torch.empty_like(full.lo), full.channels)
        outs = [out.hi] + ([out.lo] if out.lo is not None else [])
    _check_counts(cuda, lambda dyn: ops.conv_forward(xp, wp, pad, relu=relu, out_f32=f32, dyn=dyn, out=out),
                  outs, full_t, box_n, CAP, f"{name} box_n={box_n}")


# -------------------------------------------------------------------------------------------------------- pooling
def _bf16_exact(a):
    return torch.from_numpy(a).bfloat16().float().numpy()


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("mode", ["MAX", "AVE"])
@pytest.mark.parametrize("k,s", [(2, 1), (2, 2)])
@pytest.mark.parametrize("hw", [6, 8])
def test_pool_device_rows(cuda, k, s, mode, hw, split):
    """The cascade nets pool the ROIAlign grid with AVE 2/1 behind BoxOutput; 2/2 is the ROI-side MAX form."""
    from mscnn_b200 import capi, ops
    rng = np.random.default_rng(41 + hw)
    x = _bf16_exact(rng.standard_normal((CAP, 64, hw, hw)).astype(np.float32))
    ref = port.pool(x, k, s, 0, mode)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    m = capi.POOL_MAX if mode == "MAX" else capi.POOL_AVE
    full = ops.pool_forward(xp, k, s, m)
    got = ops.planes_to_nchw(full).cpu().numpy()
    assert got.shape == ref.shape
    if mode == "MAX":
        assert np.array_equal(got, ref)
    else:
        np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)
    out = ops.Planes(torch.empty_like(full.hi), None if full.lo is None else torch.empty_like(full.lo), full.channels)
    outs = [out.hi] + ([out.lo] if split else [])
    full_t = [full.hi] + ([full.lo] if split else [])
    _check_counts(cuda, lambda dyn: ops.pool_forward(xp, k, s, m, dyn=dyn, out=out), outs, full_t, 1, CAP,
                  f"pool {k}/{s} {mode}")


def _special_rois(rng, n, img_w, img_h, r):
    """The ROI mix of test_detect_gpu.test_roi_pool_parity: random boxes plus the dummy, a malformed, an outside and a
    half-pixel ROI."""
    x1 = rng.uniform(-20, img_w, r); y1 = rng.uniform(-20, img_h, r)
    bw = rng.uniform(1, 300, r); bh = rng.uniform(1, 200, r)
    rois = np.stack([rng.integers(0, n, r), x1, y1, x1 + bw, y1 + bh], axis=1).astype(np.float32)
    rois[0] = [0, 1, 1, 10, 10]
    rois[1] = [1, 50, 40, 30, 20]
    rois[2] = [0, img_w + 100, img_h + 100, img_w + 200, img_h + 200]
    rois[3] = [1, 3.5, 4.5, 4.5, 5.5]
    return rois


ROI_CAP = 64
PAD_RATIOS = (0.0, 0.25, 0.5, 1.0)
PERMS = {1: [0], 2: [1, 0], 3: [2, 0, 1], 4: [2, 0, 3, 1]}   # slot of variant i in the output
SPARE = 64                                                     # leading channels no variant may touch


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("nv", [1, 2, 3, 4])
@pytest.mark.parametrize("c", [64, 192, 384, 512, 768])
def test_roi_pool_multi_device_rows(cuda, c, nv, split):
    """Object and context windows in one launch, each at its own concat offset.  C covers lanes with one channel group
    (64), mixed paired-group lanes (192, 384), every lane paired (512, the conv4_3 case) and a second lane pass (768)."""
    from mscnn_b200 import ops
    rng = np.random.default_rng(50 + c + nv)
    n, h, w, scale, pooled = 2, 24, 80, 0.125, 7
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    rois = _special_rois(rng, n, w / scale, h / scale, ROI_CAP)
    ratios = PAD_RATIOS[:nv]
    offs = [SPARE + PERMS[nv][i] * c for i in range(nv)]
    ctot = SPARE + nv * c
    by_slot = sorted(range(nv), key=lambda i: offs[i])
    ref = port.concat_channels(*[port.roi_pool(x, rois, pooled, pooled, scale, ratios[i]) for i in by_slot])
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    dr = torch.from_numpy(rois).to(cuda)

    def planes():
        hi = torch.empty((ROI_CAP, pooled, pooled, ctot), dtype=torch.bfloat16, device=cuda)
        p = ops.Planes(hi, torch.empty_like(hi) if split else None, ctot)
        for t in [p.hi] + ([p.lo] if split else []):
            _fill(t)
        return p

    full = ops.roi_pool_multi_forward(xp, dr, ROI_CAP, pooled, scale, ratios, offs, out=planes(), out_channels=ctot)
    full_t = [full.hi] + ([full.lo] if split else [])
    for t in full_t:
        assert bool((_bits(t[..., :SPARE]) == SENT_BF16).all()), "the spare channels were written"
    got = ops.planes_to_nchw(full).cpu().numpy()[:, SPARE:]
    assert np.array_equal(got, ref)
    out = planes()
    outs = [out.hi] + ([out.lo] if split else [])
    _check_counts(cuda, lambda dyn: ops.roi_pool_multi_forward(xp, dr, ROI_CAP, pooled, scale, ratios, offs, out=out,
                                                               out_channels=ctot, dyn=dyn),
                  outs, full_t, 1, ROI_CAP, f"roi_pool C={c} variants={nv}")


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_roi_align_device_rows(cuda, split):
    """ROIAlign at channel offset C of a 2C-wide output; the first C channels keep their sentinel."""
    from mscnn_b200 import ops
    rng = np.random.default_rng(61)
    n, c, h, w, scale, pad_ratio, pooled = 2, 128, 24, 40, 0.125, 0.25, 5
    x = _bf16_exact(rng.standard_normal((n, c, h, w)).astype(np.float32))
    cap = 150
    rois = _special_rois(rng, n, w / scale, h / scale, cap)
    ref = port.roi_align(x, rois, pooled, pooled, scale, pad_ratio)
    xp = ops.nchw_to_planes(torch.from_numpy(x).to(cuda), split)
    dr = torch.from_numpy(rois).to(cuda)

    def planes():
        hi = torch.empty((cap, pooled + 1, pooled + 1, 2 * c), dtype=torch.bfloat16, device=cuda)
        p = ops.Planes(hi, torch.empty_like(hi) if split else None, 2 * c)
        for t in [p.hi] + ([p.lo] if split else []):
            _fill(t)
        return p

    full = ops.roi_align_forward(xp, dr, cap, pooled, scale, pad_ratio, out=planes(), channel_offset=c,
                                 out_channels=2 * c)
    full_t = [full.hi] + ([full.lo] if split else [])
    for t in full_t:
        assert bool((_bits(t[..., :c]) == SENT_BF16).all()), "the other half was written"
    got = ops.planes_to_nchw(full).cpu().numpy()[:, c:]
    np.testing.assert_allclose(got, ref, rtol=2.0 ** -8 if not split else 2e-5, atol=1e-6)
    assert np.array_equal(got == 0, ref == 0)
    out = planes()
    outs = [out.hi] + ([out.lo] if split else [])
    _check_counts(cuda, lambda dyn: ops.roi_align_forward(xp, dr, cap, pooled, scale, pad_ratio, out=out,
                                                          channel_offset=c, out_channels=2 * c, dyn=dyn),
                  outs, full_t, 1, cap, "roi_align")
