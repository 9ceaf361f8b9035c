"""The plane kernels between two convolutions (Pooling, global pooling, ROIPooling with its fused Concat, ROIAlign and the
depthwise Deconvolution) on inputs whose lo plane is live, against the reference bit for bit.

Method, for every kernel: fp32 NCHW inputs from faithful_planes_ref.faithful_input (>= 90 % of the elements with a
non-zero lo; hi ties inside windows whose lo decides the maximum; lo of the opposite sign to hi; lo exactly half an ulp
of hi) are split into planes by mscnn_nchw_f32_to_planes.  The reference runs on the value the planes hold,
float(hi) + float(lo) (exact in fp32, read back with planes_to_nchw), and its fp32 result r is rounded as store8 rounds:
hi' = bf16_rn(r), lo' = bf16_rn(r - hi').  The kernel's output must equal hi' + lo' bit for bit; on the plain bf16 path
(no lo plane) the input is hi alone and the output bf16_rn(r).

The one exception is global AVE pooling, which sums in its own fixed order (global_pool_kernel): it is held bit for bit
to a restatement of that order, and to the exact mean within (HW - 1) 2^-24 mean|x| plus the rounding of the division and
of the output's storage.  Where a maximum is compared with the reference's `if (x > max)` under another order or with
fmaxf (ROIPooling, global MAX), +0 and -0 compare equal; every other bit must match.

The last tests run the shipped nets with synthetic weights in both precisions and hold every Pooling, ROIPooling (with
its fused Concat), ROIAlign and depthwise Deconvolution layer to the reference applied to the layer's own bottom blobs."""
import os

import numpy as np
import pytest
import torch

import faithful_planes_ref as F
from conv_geometry_ref import pool as pool_rect
from deconv_ref import depthwise_col2im_f32
from oracle import port
from test_conv_geometry_gpu import POOLS
from test_deconv_gpu import DW_CASES
from test_detect_gpu import POOL_CASES
from test_device_rows_gpu import SENT_BF16, _bits, _fill
from test_unfused_gpu import _unstored_blobs

pytestmark = pytest.mark.gpu
KINDS = ("signed", "relu")
SPLITS = dict(argvalues=[True, False], ids=["split", "bf16"])


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _f32bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _upload(cuda, x, split):
    """Planes of x and the fp32 value they hold."""
    from mscnn_b200 import ops
    xp = ops.nchw_to_planes(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(cuda), split)
    return xp, _read(xp)


def _read(p):
    from mscnn_b200 import ops
    return ops.planes_to_nchw(p).cpu().numpy()


def _exact(got, r, split, what, signed_zero=True):
    """got == store8's rounding of the reference's fp32 result r, bit for bit (signed_zero=False: +0 == -0)."""
    want = F.stored(r, split)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    same = _f32bits(got) == _f32bits(want)
    if not signed_zero:
        same |= (got == 0) & (want == 0)
    if not same.all():
        bad = np.argwhere(~same)
        msg = [f"{what}: {len(bad)}/{got.size} elements differ, first at {bad[:6].tolist()}"]
        for i in bad[:4]:
            t = tuple(i)
            msg.append(f"  at {t}: got {got[t]!r} want {want[t]!r} (reference fp32 {r[t]!r})")
        pytest.fail("\n".join(msg))


def _sentinel_planes(cuda, shape, split):
    from mscnn_b200 import ops
    hi = torch.empty(shape, dtype=torch.bfloat16, device=cuda)
    p = ops.Planes(hi, torch.empty_like(hi) if split else None, shape[-1])
    for t in [p.hi] + ([p.lo] if split else []):
        _fill(t)
    return p


def _untouched(p, what, rows=slice(None), channels=slice(None)):
    for t in [p.hi] + ([p.lo] if p.lo is not None else []):
        assert bool((_bits(t[rows][..., channels]) == SENT_BF16).all()), f"{what}: written outside its rows / channels"


# ------------------------------------------------------------------------------------------------------------ Pooling
POOL_GEOMS = ([(f"{m}-{h}x{w}-k{k}s{s}", (m,), h, w, k, s, 0) for m, h, w, k, s in POOL_CASES]
              + [(name, ("MAX", "AVE"), h, w, k, s, p) for name, h, w, k, s, p in POOLS])


def _pool_ref(x, k, s, p, mode):
    if all(isinstance(v, int) for v in (k, s, p)):
        return port.pool(x, k, s, p, mode)
    return pool_rect(x, _pair(k), _pair(s), _pair(p), mode)


@pytest.mark.parametrize("split", **SPLITS)
@pytest.mark.parametrize("case", POOL_GEOMS, ids=[c[0] for c in POOL_GEOMS])
def test_pool_kernel(cuda, case, split):
    """MAX and AVE on the geometries of test_pool_parity and test_pool_geometry_parity (odd sizes, stride 1, 3/2,
    padding, rectangular windows, the ceil-mode decrement).  AVE divides by the window clipped to the padded extent."""
    from mscnn_b200 import capi, ops
    name, modes, h, w, k, s, p = case
    rng = np.random.default_rng(100 + h * w)
    for kind in KINDS:
        xp, rep = _upload(cuda, F.faithful_input(rng, (2, 64, h, w), kind), split)
        for mode in modes:
            out = ops.pool_forward(xp, k, s, capi.POOL_MAX if mode == "MAX" else capi.POOL_AVE, pad=p)
            # numpy's max (the rectangular restatement) may pick either zero of a +0 / -0 tie
            strict = mode == "AVE" or all(isinstance(v, int) for v in (k, s, p))
            _exact(_read(out), _pool_ref(rep, k, s, p, mode), split, f"{name} {mode} {kind}", signed_zero=strict)


@pytest.mark.parametrize("split", **SPLITS)
@pytest.mark.parametrize("mode", ["MAX", "AVE"])
@pytest.mark.parametrize("k,s,p", [(2, 1, 0), (2, 2, 0), ((3, 2), (2, 1), (1, 0))], ids=["k2s1", "k2s2", "k3x2s2x1p1x0"])
def test_pool_kernel_device_rows(cuda, k, s, p, mode, split):
    """The dyn-row form at a device count below N: the images below it exact, the rest keep the NaN sentinel."""
    from mscnn_b200 import capi, ops
    n, count = 40, 27
    rng = np.random.default_rng(7)
    xp, rep = _upload(cuda, F.faithful_input(rng, (n, 64, 6, 6), "relu"), split)
    m = capi.POOL_MAX if mode == "MAX" else capi.POOL_AVE
    shape = ops.pool_forward(xp, k, s, m, pad=p).shape
    out = _sentinel_planes(cuda, shape, split)
    ops.pool_forward(xp, k, s, m, dyn=torch.tensor([count], dtype=torch.int32, device=cuda), out=out, pad=p)
    _exact(_read(out)[:count], _pool_ref(rep[:count], k, s, p, mode), split, f"pool {mode} dyn")
    _untouched(out, "pool dyn", rows=slice(count, None))


GLOBAL_SHAPES = [(2, 64, 4, 8), (2, 264, 9, 11), (2, 512, 24, 80), (1, 64, 50, 80), (2, 512, 33, 1), (1, 264, 61, 63)]


@pytest.mark.parametrize("split", **SPLITS)
@pytest.mark.parametrize("shape", GLOBAL_SHAPES, ids=["x".join(map(str, s)) for s in GLOBAL_SHAPES])
def test_global_pool_kernel(cuda, shape, split):
    """One window over the whole image, HW = 32 .. 3843 (no four-pixel step, both steps, steps only): MAX exact; AVE
    bit for bit the kernel's stated order and within (HW - 1) 2^-24 mean|x| (+ division and storage) of the exact
    mean."""
    from mscnn_b200 import capi, ops
    n, c, h, w = shape
    rng = np.random.default_rng(200 + h * w)
    for kind in KINDS:
        xp, rep = _upload(cuda, F.faithful_input(rng, shape, kind), split)
        got = _read(ops.pool_forward(xp, None, 1, capi.POOL_MAX))
        _exact(got, rep.max(axis=(2, 3), keepdims=True), split, f"global MAX {kind}", signed_zero=False)
        got = _read(ops.pool_forward(xp, None, 1, capi.POOL_AVE))
        _exact(got, F.global_ave_kernel_order(rep), split, f"global AVE {kind} (kernel order)")
        x64 = rep.astype(np.float64)
        exact = x64.mean(axis=(2, 3), keepdims=True)
        bound = ((h * w - 1) * 2.0 ** -24 * np.abs(x64).mean(axis=(2, 3), keepdims=True) + 2.0 ** -24 * np.abs(exact)
                 + (2.0 ** -16 if split else 2.0 ** -8) * np.abs(got))
        err = np.abs(got - exact)
        assert bool((err <= bound).all()), (kind, float((err / bound).max()))


# --------------------------------------------------------------------------------------------------------- ROIPooling
ROI_BINS = [(7, 7), (5, 5), (8, 4), (1, 7)]
SPARE = 64


@pytest.mark.parametrize("split", **SPLITS)
@pytest.mark.parametrize("c", [64, 256, 512])
@pytest.mark.parametrize("bins", ROI_BINS, ids=[f"{a}x{b}" for a, b in ROI_BINS])
def test_roi_pool_kernel(cuda, bins, c, split):
    """C = 64 (one group per lane), 256 (half of the lanes pool a second group: DUAL), 512 (every lane DUAL); windows of
    odd and even pixel count (the odd-pixel tail step with and without), empty bins and the edge ROIs; scales 1/8 and
    1/4.  The fused org || ctx form: pad_ratio 0 and 0.25 in one launch at channel offsets 64 + C and 64 of a
    64 + 2C-wide output, with a device ROI count below R; then the one-variant entry."""
    from mscnn_b200 import ops
    n, h, w, r = 2, 24, 40, 96
    count = r - 7
    ph, pw = bins
    rng = np.random.default_rng(300 + c + ph * 10 + pw)
    dyn = torch.tensor([count], dtype=torch.int32, device=cuda)
    for kind in KINDS:
        xp, rep = _upload(cuda, F.faithful_input(rng, (n, c, h, w), kind), split)
        for scale in (0.125, 0.25):
            rois = F.special_rois(rng, n, w / scale, h / scale, r)
            npx = np.concatenate([F.roi_pool_windows(rois[:count], h, w, ph, pw, scale, pr).ravel() for pr in (0, .25)])
            assert (npx == 0).any() and (npx % 2 == 1).any() and ((npx > 0) & (npx % 2 == 0)).any()
            dr = torch.from_numpy(rois).to(cuda)
            ref = {pr: port.roi_pool(rep, rois[:count], ph, pw, scale, pr) for pr in (0.0, 0.25)}
            what = f"roi_pool {kind} scale {scale}"
            ctot = SPARE + 2 * c
            out = _sentinel_planes(cuda, (r, ph, pw, ctot), split)
            ops.roi_pool_multi_forward(xp, dr, r, bins, scale, [0.0, 0.25], [SPARE + c, SPARE], out=out,
                                       out_channels=ctot, dyn=dyn)
            got = _read(out)[:count]
            _exact(got[:, SPARE + c:], ref[0.0], split, what + " org", signed_zero=False)
            _exact(got[:, SPARE:SPARE + c], ref[0.25], split, what + " ctx", signed_zero=False)
            _untouched(out, what, rows=slice(count, None))
            _untouched(out, what, channels=slice(0, SPARE))
            single = ops.roi_pool_forward(xp, dr, count, bins, scale, 0.25)
            _exact(_read(single), ref[0.25], split, what + " one variant", signed_zero=False)


# ----------------------------------------------------------------------------------------------------------- ROIAlign
ALIGN_BINS = [(5, 5), (7, 7), (4, 7), (8, 4)]


@pytest.mark.parametrize("split", **SPLITS)
@pytest.mark.parametrize("bins", ALIGN_BINS, ids=[f"{a}x{b}" for a, b in ALIGN_BINS])
def test_roi_align_kernel(cuda, bins, split):
    """The malformed, outside, sub-pixel and full-map ROIs among random ones, scales 1/8 and 1/4, pad_ratio 0 and 0.25,
    written at channel offset C of a 2C-wide output with a device ROI count below R."""
    from mscnn_b200 import ops
    n, c, h, w, r = 2, 128, 24, 40, 80
    count = r - 5
    ph, pw = bins
    rng = np.random.default_rng(400 + ph * 10 + pw)
    dyn = torch.tensor([count], dtype=torch.int32, device=cuda)
    for kind in KINDS:
        xp, rep = _upload(cuda, F.faithful_input(rng, (n, c, h, w), kind), split)
        for scale in (0.125, 0.25):
            rois = F.special_rois(rng, n, w / scale, h / scale, r)
            dr = torch.from_numpy(rois).to(cuda)
            for pr in (0.0, 0.25):
                what = f"roi_align {kind} scale {scale} pad_ratio {pr}"
                ref = port.roi_align(rep, rois[:count], ph, pw, scale, pr)
                assert not ref[1].any() and not ref[2].any()                       # malformed, outside: zeros
                out = _sentinel_planes(cuda, (r, ph + 1, pw + 1, 2 * c), split)
                ops.roi_align_forward(xp, dr, r, bins, scale, pr, out=out, channel_offset=c, out_channels=2 * c, dyn=dyn)
                _exact(_read(out)[:count, c:], ref, split, what)
                _untouched(out, what, rows=slice(count, None))
                _untouched(out, what, channels=slice(0, c))


# --------------------------------------------------------------------------------------------- depthwise Deconvolution
@pytest.mark.parametrize("split", **SPLITS)
def test_deconv2x_kernel(cuda, split):
    """deconv_depthwise_kernel<4, 2, 1>, the -2x nets' layer; C = 72 leaves a padded tail of channels."""
    from mscnn_b200 import ops
    rng = np.random.default_rng(500)
    c = 72
    wt = rng.standard_normal((c, 1, 4, 4)).astype(np.float32)
    for kind in KINDS:
        xp, rep = _upload(cuda, F.faithful_input(rng, (2, c, 9, 15), kind), split)
        got = _read(ops.deconv2x_forward(xp, torch.from_numpy(wt).to(cuda)))
        _exact(got, depthwise_col2im_f32(rep, wt, None, 2, 1), split, f"deconv2x {kind}")


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("split", **SPLITS)
@pytest.mark.parametrize("case", DW_CASES, ids=[c[0] for c in DW_CASES])
def test_depthwise_kernel(cuda, case, split, bias):
    """The general deconv_depthwise_kernel on the geometries of test_depthwise_parity (bilinear_2x takes <4, 2, 1>)."""
    from mscnn_b200 import ops
    name, c, h, w, k, stride, pad, dil = case
    rng = np.random.default_rng(600 + c + h * w)
    wt = rng.standard_normal((c, 1) + _pair(k)).astype(np.float32)
    b = rng.standard_normal(c).astype(np.float32) if bias else None
    for kind in KINDS:
        xp, rep = _upload(cuda, F.faithful_input(rng, (2, c, h, w), kind), split)
        out = ops.deconv_depthwise_forward(xp, torch.from_numpy(wt).to(cuda),
                                           None if b is None else torch.from_numpy(b).to(cuda), stride, pad, dil)
        _exact(_read(out), depthwise_col2im_f32(rep, wt, b, stride, pad, dil), split, f"{name} {kind}")


# ---------------------------------------------------------------------------------------- the layers inside live nets
def _layer_params(net):
    """name -> (bottoms, tops, fields) from the net's layer parameter strings; a bottom that a Split layer copied is
    named by the blob it copies."""
    out, alias = {}, {}
    for s, typ in zip(net.layer_param_strings(), net.layer_types):
        parts = s.split("|")
        fields = dict(p.split(":", 1) for p in parts[2:] if ":" in p and not p.startswith(("b:", "t:")))
        bottoms = [alias.get(p[2:], p[2:]) for p in parts if p.startswith("b:")]
        tops = [p[2:] for p in parts if p.startswith("t:")]
        if typ == "Split":
            alias.update((t, bottoms[0]) for t in tops)
        out[parts[0]] = (bottoms, tops, fields)
    return out


def _rows(r):
    """The ROI rows a layer check compares: all of a small set, else the first 32 and 64 spread over the rest."""
    return np.arange(r) if r <= 96 else np.unique(np.concatenate([np.arange(32), np.linspace(0, r - 1, 64).astype(int)]))


def _roi_ref(net, params, layer, rows):
    bottoms, _, f = params[layer]
    ph, pw, scale, pr = f["roi"].split(",")
    x = net.blob(bottoms[0])
    rois = net.blob(bottoms[1]).reshape(-1, 5)[rows]
    fn = port.roi_align if net.layer_types[net.layer_names.index(layer)] == "ROIAlign" else port.roi_pool
    return fn(x, rois, int(ph), int(pw), float(np.float32(scale)), float(np.float32(pr)))


def _check_net_layers(net, split, unstored, only=None):
    """Every Pooling, ROIPooling (or the Concat it writes into), ROIAlign and depthwise Deconvolution layer whose bottom
    blobs are stored, against the reference on those blobs.  Returns (checked, Pooling layers left for a net without
    pool fusion)."""
    params = _layer_params(net)
    producer = {params[n][1][0]: n for n, t in zip(net.layer_names, net.layer_types) if t in ("ROIPooling", "ROIAlign")}
    checked, pending = [], []
    for name, typ in zip(net.layer_names, net.layer_types):
        if only is not None and name not in only:
            continue
        bottoms, tops, f = params[name]
        what = f"{name} ({typ}, {'split' if split else 'bf16'})"
        if typ == "Pooling":
            if bottoms[0] in unstored:
                pending.append(name)
                continue
            mode, k, s, p = (int(v) for v in f["pool"].split(","))
            x = net.blob(bottoms[0])
            rows = _rows(x.shape[0])
            mode = "MAX" if mode == 0 else "AVE"
            _exact(net.blob(tops[0])[rows], port.pool(x[rows], k, s, p, mode), split, what)
        elif typ in ("ROIPooling", "ROIAlign"):
            if tops[0] in unstored:
                continue                                     # written into its Concat: checked there
            rows = _rows(net.blob(bottoms[1]).reshape(-1, 5).shape[0])
            _exact(net.blob(tops[0])[rows], _roi_ref(net, params, name, rows), split, what, signed_zero=typ != "ROIPooling")
        elif typ == "Concat" and all(producer.get(b) and params[producer[b]][0][1] == params[producer[bottoms[0]]][0][1]
                                     for b in bottoms):
            first = params[producer[bottoms[0]]][0][1]
            rows = _rows(net.blob(first).reshape(-1, 5).shape[0])
            ref = np.concatenate([_roi_ref(net, params, producer[b], rows) for b in bottoms], axis=1)
            _exact(net.blob(tops[0])[rows], ref, split, what, signed_zero=False)
        elif typ == "Deconvolution":
            conv = f["conv"].split(",")
            num_output, bias_term, group = int(conv[0]), conv[1] in ("1", "true"), int(conv[2])
            x = net.blob(bottoms[0])
            if not (group == num_output == x.shape[1]):
                continue
            stride = int(next((v[1:] for v in conv[3:] if v.startswith("s")), 1))
            pad = int(next((v[1:] for v in conv[3:] if v.startswith("p")), 0))
            b = net.param(name, 1) if bias_term else None
            _exact(net.blob(tops[0]), depthwise_col2im_f32(x, net.param(name, 0), b, stride, pad), split, what)
        else:
            continue
        checked.append(name)
    return checked, pending


def _caltech():
    import re
    from test_pedestrian_nets_gpu import _deploy
    text, k = re.subn(r"max_nms_num: \d+", "max_nms_num: 300", _deploy("caltech/mscnn-7s-720", 2, 240, 320))
    assert k == 1
    return text


def _models(fn, *args):
    def make():                      # at most 300 proposals per image keep the ROI blobs small
        from mscnn_b200 import models
        return getattr(models, fn)(*args, batch=2, max_nms_num=300)
    return make


LIVE_NETS = [
    # name, prototxt, input h, w, the layers that must be checked
    ("kitti_8s_192x640", _models("kitti", 192, 640, 8, False), 192, 640,
     {"pool1", "pool2", "pool3", "pool4", "pool5", "pool6", "roi_pool"}),
    ("kitti_7s_2x_96x320", _models("kitti", 96, 320, 7, True), 96, 320, {"pool4", "conv4_3_2x", "roi_pool"}),
    ("wider_12s_2x_128x192", _models("widerface", 128, 192), 128, 192, {"pool6", "conv4_3_2x", "roi_pool"}),
    ("kitti_cascade_96x320", _models("kitti_cascade", 96, 320), 96, 320,
     {"conv4_3_2x", "roi_pool", "roi_pool_2nd", "roi_pool_3rd"}),
    ("wider_cascade_128x192", _models("widerface_cascade", 128, 192), 128, 192,
     {"pool6", "roi_grid_org", "roi_grid_ctx_3rd", "roi_pool_org", "roi_pool_ctx_2nd", "roi_pool_org_3rd"}),
    ("caltech_7s_240x320", _caltech, 240, 320, {"pool1", "pool6", "roi_pool"}),
]


@pytest.mark.parametrize("case", LIVE_NETS, ids=[c[0] for c in LIVE_NETS])
def test_net_plane_layers_are_exact(cuda, case):
    """After one forward with synthetic weights, in the fp32-faithful and the bf16 precision: each such layer's top
    against the reference on its bottom blob(s) and the net's own rois blob, bit for bit.  Pooling layers folded into
    their convolution's epilogue (no stored bottom) are checked in the same net built without pool fusion, which
    test_pool_fusion_is_bit_identical holds to the fused one."""
    from mscnn_b200 import net as mnet, synth
    name, make, h, w, must = case
    proto = make()
    images = synth.make_images(2, h, w)
    weights = None
    try:
        for precision in ("fp32", "bf16"):
            mnet.set_precision(precision)
            net = mnet.Net(proto)
            if weights is None:
                weights = synth.make_weights(net.layers())
            net.set_params(weights)
            net.forward(data=images)
            assert net.num_proposals() > 0
            checked, pending = _check_net_layers(net, precision == "fp32", _unstored_blobs(net))
            del net
            if pending:
                os.environ["MSCNN_NO_POOL_FUSION"] = "1"
                try:
                    flat = mnet.Net(proto)
                finally:
                    os.environ.pop("MSCNN_NO_POOL_FUSION", None)
                flat.set_params(weights)
                flat.set_input("data", images)
                flat.forward_only(end=pending[-1])
                done, left = _check_net_layers(flat, precision == "fp32", _unstored_blobs(flat), only=set(pending))
                assert not left and sorted(done) == sorted(pending), (pending, done)
                checked += done
                del flat
            assert must <= set(checked), (precision, sorted(must - set(checked)))
    finally:
        mnet.set_precision("fp32")
