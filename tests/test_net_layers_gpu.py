"""Every layer of every shipped architecture, inside a live net, against a reference applied to the layer's own bottom
blobs, in the fp32-faithful and the plain bf16 precision.

One net per architecture (tests/net_layers_ref.CASES) is built from the shipped deploy file with its input set to
2 x 3 x H x W at the size its fixtures run (KITTI 192x640, Caltech 240x320, CityPersons 192x384, WIDER FACE 128x192),
with synth.make_weights and synth.make_images and the shipped BoxOutput parameters; then kitti_car/mscnn-8s-768 at
100x324 (odd extents: pool3 runs itself, partial tiles in H and W) and widerface/mscnn-12s-2x reshaped live from 128x192
to 160x96 and back, with a forward and the full check after each reshape and no weight re-pack.

After one forward, each layer net_layers_ref.classify calls COMPUTE is checked here:
* Convolution and InnerProduct, every element of every image and every ROI row, against an fp64 reference r on the
  device: F.conv2d with the layer's pad, stride, dilation and group read from the prototxt (InnerProduct: the bottom
  flattened in Caffe's C, H, W order times W^T), plus the bias, rectified when an in-place ReLU reads the top.  The
  input is the bottom blob as the layer read it (fp32-faithful: hi + lo, exact in fp32, and the fp32 `data` for conv1_1;
  bf16: the hi plane, bf16_rn(data) for conv1_1), the weights fp32 (fp32-faithful) or bf16_rn(W) (bf16).  A top whose
  un-pooled planes are never stored is held through its pooled top, to the 2x2/2 MAX of r.  The bars are
  net_layers_ref.bar: |got - r| <= rel |r| + abs rms(r), each from the kernel-level test that measured it; every layer's
  worst |got - r| / bar is printed.
* BoxOutput against oracle.port.box_output on the net's own LFCN blobs, with the parameters of the layer's box: and reg:
  fields (field_w / field_h, downsample rates, thresholds, caps, bbox normalisation): the per-image counts against
  num_proposals(i), the image and score columns bit for bit, the box corners bit for bit except on the few rows (at most
  one in 200) where glibc's expf, which the reference calls, is not the correctly rounded exp the device computes:
  there within one ulp of the box extent plus one of the corner.
* DecodeBBox bit for bit against net_layers_ref.decode_bbox_f32 (which agrees with oracle.port.decode_bbox within one
  ulp of the exp-derived terms), Softmax and Eltwise bit for bit against oracle.port, a plain Concat against the bytes of
  its bottoms.
The PLANE layers (Pooling, ROIPooling, ROIAlign, depthwise Deconvolution) are checked bit for bit by
test_faithful_planes_gpu._check_net_layers on the same net, the Pooling layers folded into a convolution on the same
net built with MSCNN_NO_POOL_FUSION=1.  The checked layers must be exactly the ones classify does not call IDENTITY."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import net_layers_ref as R

pytestmark = pytest.mark.gpu
ROW_CHUNK = 512                  # ROI rows per fp64 reference convolution


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _exact(got, ref, what):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bad = np.argwhere(_bits(got) != _bits(ref))
    if len(bad):
        t = tuple(bad[0])
        pytest.fail(f"{what}: {len(bad)}/{got.size} elements differ, first at {bad[:6].tolist()}: got {got[t]!r} want "
                    f"{ref[t]!r}")


class LayerCheck:
    """The COMPUTE checks of one net after a forward."""

    def __init__(self, net, text, key, split, cuda):
        self.net, self.split, self.cuda = net, split, cuda
        self.params = R.layer_params(net)
        self.proto = R.prototxt_layers(text)
        self.classes = R.classify(net, text, key)
        self.rectified = R.rectified_tops(net)
        self.unstored = R._unstored_blobs(net)
        self.worst = {}
        self.box_rows_off = 0

    def _dev(self, a, rounded=True):
        """numpy fp32 -> device fp32, bf16_rn-rounded in the bf16 precision."""
        t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(self.cuda)
        return t.bfloat16().float() if rounded and not self.split else t

    def _compare(self, name, got, r, rms, k):
        rel, ab = R.bar(self.split, k)
        got = torch.from_numpy(np.ascontiguousarray(got)).to(self.cuda).double().reshape(r.shape)
        err = (got - r).abs()
        lim = rel * r.abs() + ab * rms
        ratio = float((err / lim).max())
        self.worst[name] = ratio
        if ratio > 1:
            idx = (err > lim).nonzero()
            t = tuple(idx[0].tolist())
            pytest.fail(f"{name} ({'split' if self.split else 'bf16'}, K={k}, bar {rel:g} |r| + {ab:g} rms): "
                        f"{idx.shape[0]}/{err.numel()} elements over, worst {ratio:.3g} x the bar; distinct bad indices "
                        f"per dim {[idx[:, d].unique()[:10].tolist() for d in range(idx.shape[1])]}; at {t} got "
                        f"{float(got[t]):.7g} ref {float(r[t]):.7g} (rms {rms:.4g})")

    def conv(self, name):
        net, (bottoms, tops, _) = self.net, self.params[name]
        kh, kw, ph, pw, sh, sw, dh, dw, group = R.conv_geometry(self.proto[name])
        x = self._dev(net.blob(bottoms[0]))
        w = self._dev(net.param(name, 0)).double()
        b = self._dev(net.param(name, 1), rounded=False).double() if len(net.param_shapes(name)) > 1 else None
        r = torch.cat([F.conv2d(x[i:i + ROW_CHUNK].double(), w, b, stride=(sh, sw), padding=(ph, pw),
                                dilation=(dh, dw), groups=group) for i in range(0, x.shape[0], ROW_CHUNK)])
        del x
        if tops[0] in self.rectified:
            r = torch.relu(r)
        rms = float(r.pow(2).mean().sqrt())
        k = w.shape[1] * kh * kw
        if tops[0] in self.unstored:
            pool, = [p for p, t in zip(net.layer_names, net.layer_types)
                     if t == "Pooling" and self.params[p][0][0] == tops[0] and net.fused_producer(p) == name]
            assert self.params[pool][2]["pool"] == "0,2,2,0", (name, pool)
            self._compare(f"{name} (pooled: {pool})", net.blob(self.params[pool][1][0]), F.max_pool2d(r, 2, 2), rms, k)
        else:
            self._compare(name, net.blob(tops[0]), r, rms, k)

    def inner_product(self, name):
        net, (bottoms, tops, _) = self.net, self.params[name]
        x = self._dev(net.blob(bottoms[0]))
        x = x.reshape(x.shape[0], -1).double()                  # Caffe's (C, H, W) flattening of each row
        w = self._dev(net.param(name, 0)).double()
        r = x @ w.t()
        del x
        if len(net.param_shapes(name)) > 1:
            r = r + self._dev(net.param(name, 1), rounded=False).double()
        if tops[0] in self.rectified:
            r = torch.relu(r)
        self._compare(name, net.blob(tops[0]), r, float(r.pow(2).mean().sqrt()), w.shape[1])

    def box_output(self, name):
        from oracle import port
        from test_box_edges_gpu import _same_rows
        net, (bottoms, tops, f) = self.net, self.params[name]
        box = f["box"].split(",")
        fg, iou, nms, whr, xyr, cap, post, min_size = box[:8]
        field_w = [int(v[1:]) for v in box[8:] if v.startswith("w")]
        field_h = [int(v[1:]) for v in box[8:] if v.startswith("h")]
        rate = [int(v[1:]) for v in box[8:] if v.startswith("d")]
        mean = [float(v) for v in re.findall(r"m([^ms]+)", f["reg"])]
        std = [float(v) for v in re.findall(r"s([^ms]+)", f["reg"])]
        assert len(field_w) == len(field_h) == len(rate) == len(bottoms) and len(mean) == len(std) in (0, 4)
        maps = [net.blob(b) for b in bottoms]
        rois, scores, per, true = port.box_output(maps, field_w, field_h, rate, float(fg), float(iou), nms, float(whr),
                                                  float(xyr), float(min_size), int(cap), int(post), mean or None,
                                                  std or None)
        n = maps[0].shape[0]
        assert [net.num_proposals(i) for i in range(n)] == list(per) and net.num_proposals() == true > 0, (name, per)
        got_rois, got_scores = net.blob(tops[0]).reshape(-1, 5), net.blob(tops[1]).reshape(-1, 6)
        assert got_rois.shape == rois.shape and got_scores.shape == scores.shape
        # image and score columns bit for bit (so the ranking and every NMS decision are the reference's); the box
        # corners bit for bit except where glibc's expf, which the reference calls, and exp in fp64 rounded once, which
        # the device calls, differ in the last bit: within one ulp of the box extent plus one of the corner
        _same_rows(got_rois[:, :1], rois[:, :1])
        _same_rows(got_scores[:, [0, 5]], scores[:, [0, 5]], score_col=1)
        for got, ref in ((got_rois[:, 1:5], rois[:, 1:5]), (got_scores[:, 1:5], scores[:, 1:5])):
            extent = np.abs(ref[:, [2, 3, 2, 3]] - ref[:, [0, 1, 0, 1]]) + np.float32(1)
            bound = np.spacing(extent.astype(np.float32)) + np.spacing(np.abs(ref))
            off = _bits(got) != _bits(ref)
            assert bool((np.abs(got.astype(np.float64) - ref) <= bound).all()), (name, np.argwhere(off)[:4].tolist())
            self.box_rows_off = int(off.any(axis=1).sum())
            assert self.box_rows_off <= max(2, len(ref) // 200), (name, self.box_rows_off, len(ref))

    def decode_bbox(self, name):
        net, (bottoms, tops, f) = self.net, self.params[name]
        mean = [float(v) for v in re.findall(r"m([^ms]+)", f["reg"])] or [0.0] * 4
        std = [float(v) for v in re.findall(r"s([^ms]+)", f["reg"])] or [1.0] * 4
        pred, prior = net.blob(bottoms[0]), net.blob(bottoms[1])
        ref = R.decode_bbox_f32(pred, prior, mean, std)
        _exact(net.blob(tops[0]).reshape(-1, 5), ref, name)
        R.check_decode_against_port(ref, pred, prior, mean, std)

    def softmax(self, name):
        from oracle import port
        net, (bottoms, tops, f) = self.net, self.params[name]
        _exact(net.blob(tops[0]), port.softmax(net.blob(bottoms[0]), int(f["softmax"])), name)

    def eltwise(self, name):
        from oracle import port
        net, (bottoms, tops, f) = self.net, self.params[name]
        op = {0: "PROD", 1: "SUM", 2: "MAX"}[int(f["elt"].split(",")[0])]
        # the coefficients from the prototxt: the parameter string prints them to six digits
        coeffs = [float(v) for v in self.proto[name].get("eltwise_param.coeff", [])] or None
        _exact(net.blob(tops[0]), port.eltwise([net.blob(b) for b in bottoms], op, coeffs), name)

    def concat(self, name):
        net, (bottoms, tops, _) = self.net, self.params[name]
        _exact(net.blob(tops[0]), np.concatenate([net.blob(b) for b in bottoms], axis=1), name)

    def run(self):
        """Every COMPUTE layer; returns the names checked."""
        by_type = {"Convolution": self.conv, "InnerProduct": self.inner_product, "BoxOutput": self.box_output,
                   "DecodeBBox": self.decode_bbox, "Softmax": self.softmax, "Eltwise": self.eltwise,
                   "Concat": self.concat}
        done = []
        for name, typ in zip(self.net.layer_names, self.net.layer_types):
            if self.classes[name][0] == R.COMPUTE:
                by_type[typ](name)
                done.append(name)
        torch.cuda.empty_cache()
        return done


def _plane_layers(net, text, weights, images, split, classes):
    """test_net_plane_layers_are_exact's check on this net: _check_net_layers, then the Pooling layers it leaves
    pending on the same net built without pool fusion.  -> the PLANE layers covered."""
    from mscnn_b200 import net as mnet
    from test_faithful_planes_gpu import _check_net_layers
    unstored = R._unstored_blobs(net)
    checked, pending = _check_net_layers(net, split, unstored)
    if pending:
        os.environ["MSCNN_NO_POOL_FUSION"] = "1"
        try:
            flat = mnet.Net(text)
        finally:
            os.environ.pop("MSCNN_NO_POOL_FUSION", None)
        flat.set_params(weights)
        flat.set_input("data", images)
        flat.forward_only(end=pending[-1])
        done, left = _check_net_layers(flat, split, R._unstored_blobs(flat), only=set(pending))
        assert not left and sorted(done) == sorted(pending), (pending, done)
        checked += done
        del flat
    return R.checked_by_planes(net, classes, checked, unstored)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("case", R.CASES, ids=[c[0] for c in R.CASES])
def test_net_layers_against_reference(cuda, case, precision):
    from mscnn_b200 import capi, net as mnet, synth
    cid, key, sizes = case
    split = precision == "fp32"
    L = capi.lib()
    try:
        mnet.set_precision(precision)
        net = mnet.Net(R.deploy(key, R.BATCH, *sizes[0]))
        weights = synth.make_weights(net.layers())
        net.set_params(weights)
        for step, (h, w) in enumerate(sizes):
            text = R.deploy(key, R.BATCH, h, w)
            images = synth.make_images(R.BATCH, h, w)
            if step:
                net.reshape_input("data", R.BATCH, 3, h, w)
            packs = int(L.mscnn_weight_pack_count())
            net.forward(data=images)
            if step:
                assert int(L.mscnn_weight_pack_count()) == packs, "a live reshape re-packed weights"
            assert net.blob_shape("data") == (R.BATCH, 3, h, w)
            check = LayerCheck(net, text, key, split, cuda)
            computed = check.run()
            planes = _plane_layers(net, text, weights, images, split, check.classes)
            want = {n for n, (k, _) in check.classes.items() if k != R.IDENTITY}
            assert sorted(set(computed) | planes) == sorted(want), sorted(want ^ (set(computed) | planes))
            assert not set(computed) & planes
            worst = sorted(check.worst.items(), key=lambda kv: -kv[1])
            print(f"\n{cid} {h}x{w} {precision}: {net.num_proposals()} proposals ({check.box_rows_off} with a corner "
                  f"off by the last bit of exp), {len(computed)} computed + "
                  f"{len(planes)} plane layers checked; worst |got - r| / bar: "
                  + ", ".join(f"{n} {v:.3f}" for n, v in worst))
    finally:
        mnet.set_precision("fp32")
