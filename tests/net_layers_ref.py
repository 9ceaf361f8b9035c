"""Shared by tests/test_net_layers_cpu.py and tests/test_net_layers_gpu.py: which check each layer of a shipped net gets,
the convolution geometry read from the prototxt text, the fp64 references of the Convolution and InnerProduct layers
and their bars, and DecodeBBox restated in numpy float32.  Nothing here needs a GPU.

Each layer of a net gets exactly one check (classify):
  COMPUTE   Convolution, InnerProduct, BoxOutput, DecodeBBox, Softmax, Eltwise, and a Concat that no ROI layer
            writes into (the WIDER cascade's pooled ROIAlign grids): test_net_layers_gpu.py holds the top to a reference
            on the layer's own bottom blobs;
  PLANE     Pooling, ROIPooling (alone or through the Concat it writes), ROIAlign, depthwise Deconvolution:
            test_faithful_planes_gpu._check_net_layers holds them bit for bit;
  IDENTITY  Input, Split, Dropout (TEST phase) and a ReLU folded into its producer (the producer's check applies it).
Anything else is refused: a new layer type, a dense Deconvolution (no shipped net has one) or a Convolution whose
geometry takes none of the routes below raises Unchecked, so it cannot run unchecked."""
import re

import numpy as np

from test_fusion_cpu import EXPECTED as FUSION_PINS
from test_pedestrian_nets_gpu import _deploy as deploy     # noqa: F401  (the shipped file with its input set)
from test_unfused_gpu import _unstored_blobs                # noqa: F401

COMPUTE, PLANE, IDENTITY = "compute", "plane", "identity"


class Unchecked(Exception):
    """A layer no check covers."""


# ----------------------------------------------------------------------------------------------- the layer list
def layer_params(net):
    """name -> (bottoms, tops, fields), as test_faithful_planes_gpu._layer_params parses layer_param_strings(): a bottom
    that a Split layer copied is named by the blob it copies."""
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


def _tokens(text):
    text = re.sub(r"#[^\n]*", "", text)
    return re.findall(r'[{}]|[A-Za-z_][A-Za-z0-9_]*\s*:?|"[^"]*"|[^\s{}:"]+', text)


def prototxt_layers(text):
    """{layer name: {field: [values]}} of every `layer { }` block, nested messages flattened into "msg.field" keys."""
    toks = _tokens(text)
    layers, stack, i = {}, [], 0
    cur = None
    while i < len(toks):
        t = toks[i]
        if t == "}":
            stack.pop()
            if not stack:
                layers[cur["name"][0]] = cur
                cur = None
            i += 1
            continue
        key = t.rstrip(": \t")
        if i + 1 < len(toks) and toks[i + 1] == "{":
            if not stack and key == "layer":
                cur = {}
            stack.append(key)
            i += 2
            continue
        val = toks[i + 1].strip('"')
        if cur is not None:
            path = ".".join(stack[1:] + [key])
            cur.setdefault(path, []).append(val)
        i += 2
    return layers


def conv_geometry(fields):
    """(kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w, group) of a convolution_param, as Caffe reads it
    (base_conv_layer.cpp:27-124): kernel_h / kernel_w, pad_h / pad_w and stride_h / stride_w take precedence over the
    repeated kernel_size, pad and stride, whose one value serves both axes."""
    def get(k):
        return [int(v) for v in fields.get("convolution_param." + k, [])]

    ks, pads, strides, dils = get("kernel_size"), get("pad"), get("stride"), get("dilation")
    if get("kernel_h") or get("kernel_w"):
        kh, kw = get("kernel_h")[0], get("kernel_w")[0]
    else:
        kh, kw = ks[0], ks[-1]
    if get("pad_h") or get("pad_w"):
        ph, pw = (get("pad_h") or [0])[0], (get("pad_w") or [0])[0]
    else:
        ph = pads[0] if pads else 0
        pw = pads[1] if len(pads) > 1 else ph
    if get("stride_h") or get("stride_w"):
        sh, sw = (get("stride_h") or [1])[0], (get("stride_w") or [1])[0]
    else:
        sh = strides[0] if strides else 1
        sw = strides[1] if len(strides) > 1 else sh
    dh = dils[0] if dils else 1
    dw = dils[1] if len(dils) > 1 else dh
    return kh, kw, ph, pw, sh, sw, dh, dw, (get("group") or [1])[0]


def fused_relus(key):
    """The ReLUs test_fusion_cpu pins as folded into their producer for the shipped deploy file `key`."""
    relu = FUSION_PINS[key].split("|")[1].split()
    assert relu[0] == "relu"
    return set(relu[1:])


def rectified_tops(net):
    """Tops an in-place ReLU reads, folded into the producer or not: what the producer's top holds after a forward."""
    p = layer_params(net)
    return {p[n][0][0] for n, t in zip(net.layer_names, net.layer_types) if t == "ReLU" and p[n][0] == p[n][1]}


def conv_route(net, name, geo):
    """The route ConvolutionLayer::Forward_gpu takes for this layer (caffe_layers.cu), or Unchecked."""
    kh, kw, ph, pw, sh, sw, dh, dw, group = geo
    cout, cin = net.param_shapes(name)[0][0], net.blob_shape(layer_params(net)[name][0][0])[1]
    plain = sh == sw == dh == dw == group == 1
    rectified = layer_params(net)[name][1][0] in rectified_tops(net)
    if cin == 3 and (kh, kw, ph, pw, cout) == (3, 3, 1, 1, 64) and plain:
        return "conv1_1"
    if cout in (6, 9) and kh == kw > 1 and ph == pw and 2 * ph + 1 == kh and not rectified and cin % 64 == 0 and plain:
        return "head_taps"
    if cout <= 32:
        return "direct_f32"
    if not plain:
        raise Unchecked(f"{name}: stride {sh}x{sw}, dilation {dh}x{dw}, group {group} on the planes route")
    return "planes"


def classify(net, text, key):
    """{layer: (kind, detail)} for every layer of the net built from prototxt `text` (the shipped file `key`)."""
    params = layer_params(net)
    proto = prototxt_layers(text)
    relus = fused_relus(key)
    roi_producers = {params[n][1][0] for n, t in zip(net.layer_names, net.layer_types) if t in ("ROIPooling", "ROIAlign")}
    out = {}
    for name, typ in zip(net.layer_names, net.layer_types):
        bottoms, tops, f = params[name]
        if typ in ("Input", "Split", "Dropout"):
            out[name] = (IDENTITY, typ)
        elif typ == "ReLU":
            if name not in relus or bottoms != tops:
                raise Unchecked(f"{name}: a ReLU that is not folded into its producer")
            out[name] = (IDENTITY, "folded ReLU")
        elif typ == "Convolution":
            geo = conv_geometry(proto[name])
            wshape = net.param_shapes(name)[0]
            conv = f["conv"].split(",")
            assert wshape[2:] == geo[:2] and int(conv[0]) == wshape[0] and int(conv[2]) == geo[8], (name, wshape, geo)
            assert all(int(v[1:]) in (geo[2], geo[3]) for v in conv[3:] if v.startswith("p")), (name, conv, geo)
            out[name] = (COMPUTE, conv_route(net, name, geo))
        elif typ == "InnerProduct":
            out[name] = (COMPUTE, "fc_planes" if int(f["ip"]) > 32 else "fc_f32")
        elif typ in ("BoxOutput", "DecodeBBox", "Softmax", "Eltwise"):
            out[name] = (COMPUTE, typ)
        elif typ in ("Pooling", "ROIPooling", "ROIAlign"):
            out[name] = (PLANE, typ)
        elif typ == "Deconvolution":
            conv = f["conv"].split(",")
            if not int(conv[0]) == int(conv[2]) == net.blob_shape(bottoms[0])[1]:
                raise Unchecked(f"{name}: a dense Deconvolution")
            out[name] = (PLANE, "depthwise Deconvolution")
        elif typ == "Concat":
            out[name] = (PLANE, "ROI Concat") if all(b in roi_producers for b in bottoms) else (COMPUTE, typ)
        else:
            raise Unchecked(f"{name}: layer type {typ}")
    return out


def checked_by_planes(net, classes, plane_checked, unstored):
    """The PLANE layers _check_net_layers covered: those it returned, and each ROIPooling whose top it wrote straight
    into a Concat that was checked."""
    params = layer_params(net)
    done = set(plane_checked)
    for name, (kind, what) in classes.items():
        tops = params[name][1]
        if kind == PLANE and what == "ROIPooling" and tops[0] in unstored:
            if any(classes[c][1] == "ROI Concat" and tops[0] in params[c][0] and c in done for c in classes):
                done.add(name)
    return done


# ------------------------------------------------------------------------------------------------------- bars
# Convolution and InnerProduct, |got - r| <= rel |r| + abs rms(r), with K = Cin / group * kh * kw.  Each tier applies
# from its K upward.
#  fp32-faithful: 1e-4 (|r| + rms)                          test_conv_plan_coverage_gpu._check_values
#                 2e-4 (|r| + rms) from K = 16,384          fc6 on the 8x4 grid, test_pedestrian_layers_gpu
#                 1e-4 |r| + 5e-4 rms from K = 17,920       the 7x5 head at Cin 512 (53,760 split products),
#                                                           test_pedestrian_layers_gpu.test_conv_head_rect
#  bf16:          2^-8 |r| + 1e-5 max(1, sqrt(K / 512)) rms test_conv_plan_coverage_gpu._check_values
#                 2^-8 |r| + 1e-4 rms from K = 9,216        roi_c1 and fc6, test_pedestrian_layers_gpu
SPLIT_TIERS = [(0, 1e-4, 1e-4), (16384, 2e-4, 2e-4), (17920, 1e-4, 5e-4)]
BF16_TIERS = [(9216, 2.0 ** -8, 1e-4)]


def bar(split: bool, k: int):
    """(rel, abs in units of rms(r)) for a layer of reduction length k."""
    if split:
        return [(rel, ab) for k0, rel, ab in SPLIT_TIERS if k >= k0][-1]
    tiers = [(rel, ab) for k0, rel, ab in BF16_TIERS if k >= k0]
    return tiers[-1] if tiers else (2.0 ** -8, 1e-5 * max(1.0, (k / 512) ** 0.5))


# ------------------------------------------------------------------------------------------------- DecodeBBox
def decode_bbox_f32(bbox_pred, prior, mean, std):
    """decode_bbox_kernel (cascade.cu) restated in numpy float32: DecodeBBoxesWithPrior (math_functions.cpp:46-77) for
    class 1 (columns 4..7), every operation one fp32 rounding in the reference's order, no fused multiply-add, exp in
    fp64 rounded once.  -> [R, 5] = image, x1, y1, x2, y2."""
    f = np.float32
    q = np.ascontiguousarray(prior, dtype=f).reshape(-1, 5)
    b = np.ascontiguousarray(bbox_pred, dtype=f).reshape(len(q), -1)[:, 4:8]
    m, s = np.asarray(mean, dtype=f), np.asarray(std, dtype=f)
    with np.errstate(over="ignore"):
        pw = (q[:, 3] - q[:, 1]) + f(1)
        ph = (q[:, 4] - q[:, 2]) + f(1)
        cx = f(0.5) * (q[:, 3] + q[:, 1])
        cy = f(0.5) * (q[:, 4] + q[:, 2])
        bx = b[:, 0] * s[0] + m[0]
        by = b[:, 1] * s[1] + m[1]
        bw = b[:, 2] * s[2] + m[2]
        bh = b[:, 3] * s[3] + m[3]
        tx = bx * pw + cx
        ty = by * ph + cy
        tw = pw * np.exp(bw.astype(np.float64)).astype(f)
        th = ph * np.exp(bh.astype(np.float64)).astype(f)
        tx = tx - (tw - f(1)) / f(2)
        ty = ty - (th - f(1)) / f(2)
        return np.stack([q[:, 0], tx, ty, (tx + tw) - f(1), (ty + th) - f(1)], axis=1).astype(f)


# ------------------------------------------------------------------------------------------------- the nets run
def _family_size(key):
    """The fixture size of each family: KITTI 192x640, Caltech 240x320, CityPersons 192x384, WIDER FACE 128x192."""
    return {"kitti_car": (192, 640), "kitti_ped_cyc": (192, 640), "caltech": (240, 320), "citypersons": (192, 384),
            "widerface": (128, 192)}[key.split("/")[0]]


# One representative file per architecture (a -trainval file whose layers equal its sibling's is not run twice).
ARCHITECTURES = [
    "caltech/mscnn-7s-480", "caltech/mscnn-7s-480-2x", "caltech/mscnn-7s-720",
    "citypersons/cascade-mscnn-8s-1344-2x", "citypersons/mscnn-8s-1344-2x",
    "kitti_car/cascade-mscnn-7s-576-2x", "kitti_car/mscnn-7s-384", "kitti_car/mscnn-7s-384-2x", "kitti_car/mscnn-7s-576",
    "kitti_car/mscnn-7s-576-2x", "kitti_car/mscnn-8s-768-trainval",
    "kitti_ped_cyc/mscnn-7s-384", "kitti_ped_cyc/mscnn-7s-384-2x", "kitti_ped_cyc/mscnn-7s-576",
    "kitti_ped_cyc/mscnn-7s-576-2x", "kitti_ped_cyc/mscnn-8s-768-trainval",
    "widerface/cascade-mscnn-12s-align", "widerface/mscnn-12s-2x",
]
BATCH = 2
# (id, shipped file, the input sizes in turn: one net, reshaped live between them)
CASES = ([(k.replace("/", "-"), k, [_family_size(k)]) for k in ARCHITECTURES]
         + [("kitti_car-mscnn-8s-768-odd-100x324", "kitti_car/mscnn-8s-768-trainval", [(100, 324)]),
            ("widerface-mscnn-12s-2x-reshaped", "widerface/mscnn-12s-2x", [(128, 192), (160, 96), (128, 192)])])


def check_decode_against_port(restated, bbox_pred, prior, mean, std):
    """The restatement against oracle.port.decode_bbox (the reference's code with glibc's expf): the image column
    exactly; a coordinate within one ulp of its exp-derived width or height (expf and exp in fp64 rounded once may
    differ by one ulp there, and the subtractions carry that) plus one ulp of the coordinate itself."""
    from oracle import port
    f = np.float32
    ref = port.decode_bbox(bbox_pred, prior, mean, std)
    assert restated.shape == ref.shape and np.array_equal(restated[:, 0], ref[:, 0])
    q = np.ascontiguousarray(prior, dtype=f).reshape(-1, 5)
    b = np.ascontiguousarray(bbox_pred, dtype=f).reshape(len(q), -1)[:, 4:8]
    m, s = np.asarray(mean, dtype=f), np.asarray(std, dtype=f)
    with np.errstate(over="ignore"):
        tw = ((q[:, 3] - q[:, 1]) + f(1)) * np.exp((b[:, 2] * s[2] + m[2]).astype(np.float64)).astype(f)
        th = ((q[:, 4] - q[:, 2]) + f(1)) * np.exp((b[:, 3] * s[3] + m[3]).astype(np.float64)).astype(f)
    t = np.abs(np.stack([tw, th, tw, th], axis=1))
    bound = np.spacing(t) + np.spacing(np.abs(ref[:, 1:]))
    err = np.abs(restated[:, 1:].astype(np.float64) - ref[:, 1:])
    finite = np.isfinite(ref[:, 1:])
    assert np.array_equal(finite, np.isfinite(restated[:, 1:]))
    assert bool((err[finite] <= bound[finite]).all()), float((err[finite] / bound[finite]).max())
