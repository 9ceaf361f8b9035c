"""Shared by tests/test_conv_geometry_cpu.py, tests/test_conv_geometry_gpu.py and tests/golden/make_geometry_golden.py:
closed-form shapes, a numpy restatement of the reference's pooling with rectangular kernel / stride / pad, and the small
net that runs every new layer geometry end to end.

Reference: ConvolutionLayer::compute_output_shape (conv_layer.cpp:8-22), PoolingLayer::Reshape / Forward_cpu
(pooling_layer.cpp:79-123, :128-220)."""
import numpy as np


def conv_out(size, k, pad, stride=1, dil=1):
    return (size + 2 * pad - (dil * (k - 1) + 1)) // stride + 1


def pooled(size, k, stride, pad):
    out = -(-(size + 2 * pad - k) // stride) + 1
    if pad and (out - 1) * stride >= size + pad:      # the last window would start in the padding
        out -= 1
    return out


def pool(x, kernel, stride, pad, mode):
    """x [N, C, H, W] fp32; kernel, stride, pad = (h, w).  MAX clips the window to the image; AVE sums the clipped window
    row-major in fp32 and divides by the window clipped to the PADDED extent (pooling_layer.cpp:196-204)."""
    x = np.asarray(x, dtype=np.float32)
    n, c, h, w = x.shape
    (kh, kw), (sh, sw), (ph, pw) = kernel, stride, pad
    ho, wo = pooled(h, kh, sh, ph), pooled(w, kw, sw, pw)
    y = np.empty((n, c, ho, wo), dtype=np.float32)
    for i in range(ho):
        for j in range(wo):
            hs, ws = i * sh - ph, j * sw - pw
            he, we = min(hs + kh, h + ph), min(ws + kw, w + pw)
            size = np.float32((he - hs) * (we - ws))
            hs, ws, he, we = max(hs, 0), max(ws, 0), min(he, h), min(we, w)
            win = x[:, :, hs:he, ws:we].reshape(n, c, -1)
            if mode == "MAX":
                y[:, :, i, j] = win.max(axis=2)
            else:
                acc = np.zeros((n, c), dtype=np.float32)
                for t in range(win.shape[2]):
                    acc = acc + win[:, :, t]
                y[:, :, i, j] = acc / size
    return y


def geometry_net(h, w, batch=2):
    """A stride-2 first convolution on the image, a dilated 3x3, a grouped 3x3, a padded 3x3 / 2 MAX pool, a 1x1 with
    rectangular stride, a 2x2 / 2 MAX pool that folds into it at even extents, a rectangular AVE pool, and a global AVE
    pool feeding an InnerProduct."""
    def conv(name, bottom, cout, extra, relu=True):
        s = (f'layer {{ name: "{name}" type: "Convolution" bottom: "{bottom}" top: "{name}" '
             f'convolution_param {{ num_output: {cout} {extra} }} }}\n')
        if relu:
            s += f'layer {{ name: "relu_{name}" type: "ReLU" bottom: "{name}" top: "{name}" }}\n'
        return s

    def pool_(name, bottom, extra):
        return (f'layer {{ name: "{name}" type: "Pooling" bottom: "{bottom}" top: "{name}" '
                f'pooling_param {{ {extra} }} }}\n')

    return (f'name: "geometry"\ninput: "data"\ninput_dim: {batch} input_dim: 3 input_dim: {h} input_dim: {w}\n'
            + conv("c_stride2", "data", 64, "kernel_size: 3 pad: 1 stride: 2")
            + conv("c_dil2", "c_stride2", 128, "kernel_size: 3 pad: 2 dilation: 2")
            + conv("c_group2", "c_dil2", 128, "kernel_size: 3 pad: 1 group: 2")
            + pool_("p_pad", "c_group2", "pool: MAX kernel_size: 3 stride: 2 pad: 1")
            + conv("c_rect", "p_pad", 64, "kernel_h: 1 kernel_w: 3 pad_h: 0 pad_w: 1 stride_h: 1 stride_w: 2 dilation: 1 dilation: 1")
            + pool_("p_fold", "c_rect", "pool: MAX kernel_size: 2 stride: 2")
            + pool_("p_rect", "p_fold", "pool: AVE kernel_h: 3 kernel_w: 2 stride_h: 2 stride_w: 1 pad_h: 1 pad_w: 0")
            + pool_("p_global", "p_rect", "pool: AVE global_pooling: true")
            + 'layer { name: "fc" type: "InnerProduct" bottom: "p_global" top: "fc" inner_product_param { num_output: 10 } }\n')


GEOMETRY_BLOBS = ["c_stride2", "c_dil2", "c_group2", "p_pad", "c_rect", "p_fold", "p_rect", "p_global", "fc"]
GEOMETRY_SIZES = [(28, 44), (21, 48)]   # p_fold folds into c_rect at the first size only (odd extents at the second)
