"""Seeded synthetic inputs and weights for the MS-CNN deploy nets.

There is no network access, so neither KITTI images nor the pretrained caffemodels
(examples/kitti_car/fetch_mscnn_car_model.sh) are available; and the deploy prototxts carry no
fillers (Caffe's default is constant 0, which would make every output degenerate).  Both the
reference arm (oracle/_ref) and this framework are therefore fed from the SAME generator below,
by layer name, the way Net::CopyTrainedLayersFrom does (net.cpp:750-785).

Image    : uint8 ~ U{0..255} per BGR channel minus the mean [104,117,123]
           (examples/kitti_car/run_mscnn_detection.m:38,67-68), NCHW fp32, seed 1706 + index
           (1706 = the reference's solver random_seed).
Weights  : per-layer numpy PCG64 stream seeded with 1706 + crc32(layer name):
  * trunk / loss1_conv1 / rpn_*_conv / roi_c1 / fc6 : MSRA normal N(0, 2/fan_in), bias 0.
    The first conv (3 input channels) additionally carries a 1/64 gain so that activations are
    O(1) instead of O(100) (the image has second moment ~5.5e3).
  * LFCN_* proposal heads: class rows N(0, s_cls), box rows N(0, s_box) with
    s = target_std / sqrt(fan_in * M2_HEAD); background bias +BG_BIAS.  Calibrated once
    (tools/calibrate_synth.py) so that ~3/4 of the anchors pass fg_thr = -5, the top-2000 cap is
    hit, and the dx/dy/dw/dh clamps (box_output_layer.cpp:145-151) trigger on a few percent.
  * cls_pred* / bbox_pred* (every cascade stage): N(0, target/sqrt(K * M2_FC)), bias 0.
  * Deconvolution with a square kernel (conv4_3_2x): the exact BilinearFiller weights (include/caffe/filler.hpp:248-258),
    zero bias with bias_term; a rectangular kernel takes the MSRA rule of the trunk.
"""
from __future__ import annotations

import zlib

import numpy as np

SEED = 1706
MEAN_BGR = np.array([104.0, 117.0, 123.0], dtype=np.float32)
FIRST_CONV_GAIN = 1.0 / 64.0
M2_HEAD = 5.0       # second moment of the proposal heads' inputs under this init (measured)
M2_FC = 12.7        # second moment of fc6 outputs incl. DC component (tools/calibrate_synth.py)
CLS_STD, BOX_STD, BG_BIAS = 4.0, 0.4, 6.0
PRED_CLS_STD, PRED_BOX_STD = 2.0, 1.0


def make_images(n: int, h: int, w: int, first_index: int = 0) -> np.ndarray:
    """[n,3,h,w] fp32, BGR minus mean; image i uses seed SEED + first_index + i."""
    out = np.empty((n, 3, h, w), dtype=np.float32)
    for i in range(n):
        rng = np.random.default_rng(SEED + first_index + i)
        out[i] = rng.integers(0, 256, size=(3, h, w)).astype(np.float32) - MEAN_BGR.reshape(3, 1, 1)
    return out


def _rng(name: str) -> np.random.Generator:
    return np.random.default_rng(SEED + zlib.crc32(name.encode()))


def bilinear_kernel(k: int) -> np.ndarray:
    """BilinearFiller (filler.hpp:248-258) for a k x k filter."""
    f = int(np.ceil(k / 2.0))
    c = np.float32((2 * f - 1 - f % 2) / (2.0 * f))
    x = np.arange(k, dtype=np.float32)
    w1 = (1 - np.abs(x / np.float32(f) - c)).astype(np.float32)
    return np.outer(w1, w1).astype(np.float32)


def make_weights(layers: list[tuple[str, str, list[tuple[int, ...]]]]) -> dict[str, list[np.ndarray]]:
    """layers: (name, type, param blob shapes) in net order -> {name: [weight, bias?]} fp32."""
    out: dict[str, list[np.ndarray]] = {}
    for name, ltype, shapes in layers:
        if not shapes:
            continue
        rng = _rng(name)
        wshape = tuple(shapes[0])
        fan_in = int(np.prod(wshape[1:]))
        blobs: list[np.ndarray]
        if ltype == "Deconvolution" and wshape[-1] == wshape[-2]:
            k = wshape[-1]
            w = np.broadcast_to(bilinear_kernel(k), wshape).astype(np.float32).copy()
            blobs = [w] + [np.zeros(s, dtype=np.float32) for s in shapes[1:]]   # bias_term: zero bias
        elif ltype == "Convolution" and name.startswith("LFCN"):
            cout = wshape[0]
            cls = cout - 4
            w = rng.standard_normal(wshape).astype(np.float32)
            w[:cls] *= np.float32(CLS_STD / np.sqrt(fan_in * M2_HEAD))
            w[cls:] *= np.float32(BOX_STD / np.sqrt(fan_in * M2_HEAD))
            b = np.zeros(cout, dtype=np.float32)
            b[0] = BG_BIAS
            blobs = [w, b]
        elif ltype == "InnerProduct" and name.startswith(("cls_pred", "bbox_pred")):   # incl. cascade stages
            std = PRED_CLS_STD if name.startswith("cls_pred") else PRED_BOX_STD
            w = (rng.standard_normal(wshape) * (std / np.sqrt(fan_in * M2_FC))).astype(np.float32)
            blobs = [w, np.zeros(wshape[0], dtype=np.float32)]
        else:  # MSRA (a Deconvolution with a non-square kernel too; its bias blob is [Cout], not wshape[0])
            w = (rng.standard_normal(wshape) * np.sqrt(2.0 / fan_in)).astype(np.float32)
            if ltype == "Convolution" and wshape[1] == 3:
                w *= np.float32(FIRST_CONV_GAIN)
            blobs = [w, np.zeros(shapes[1] if len(shapes) > 1 else wshape[0], dtype=np.float32)]
        out[name] = blobs[: len(shapes)]
    return out
