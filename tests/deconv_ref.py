"""Shared by tests/test_deconv_cpu.py, tests/test_deconv_gpu.py, tests/test_faithful_planes_*.py and
tests/golden/make_deconv_golden.py: the reference's deconvolution restated in numpy (the direct scatter of col2im, and
its split by output phase into stride-1 convolutions that mscnn_deconv_forward runs; the depthwise layer in the
reference's fp32 order), the packed-weight layout, and the small net that runs every served Deconvolution geometry end
to end.

Reference: DeconvolutionLayer::compute_output_shape / Forward_cpu (deconv_layer.cpp:8-40), col2im_cpu
(util/im2col.cpp)."""
from math import gcd

import numpy as np


def deconv_out(size, k, stride=1, pad=0, dil=1):
    return stride * (size - 1) + dil * (k - 1) + 1 - 2 * pad


def axis_phase(k, s, p, d, out, r):
    """Phase r of one axis: (taps t_0 < ... < t_{m-1} reaching outputs q s + r, sub-dilation, signed pad, extent)."""
    taps = [t for t in range(k) if (r + p - t * d) % s == 0]
    ext = max(0, -(-(out - r) // s))
    pad = -((r + p - taps[-1] * d) // s) if taps else 0
    return taps, d // gcd(s, d), pad, ext


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def scatter_deconv(x, w, stride, pad, dil=1, group=1, bias=None):
    """The reference's arithmetic in float64: y[n, co, i s - p + t d] += x[n, ci, i] w[ci, co', t] over the taps, then
    the bias.  x [N, Cin, H, W], w [Cin, Cout / group, KH, KW]."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(pad), _pair(dil)
    n, cin, h, wd = x.shape
    cout_g, kh, kw = w.shape[1:]
    cin_g = cin // group
    ho, wo = deconv_out(h, kh, sh, ph, dh), deconv_out(wd, kw, sw, pw, dw)
    # the full col2im canvas with the padding, cropped at the end
    full = np.zeros((n, cout_g * group, sh * (h - 1) + dh * (kh - 1) + 1, sw * (wd - 1) + dw * (kw - 1) + 1))
    for g in range(group):
        xg = x[:, g * cin_g:(g + 1) * cin_g]
        for ky in range(kh):
            for kx in range(kw):
                contrib = np.einsum("nchw,co->nohw", xg, w[g * cin_g:(g + 1) * cin_g, :, ky, kx])
                full[:, g * cout_g:(g + 1) * cout_g, ky * dh:ky * dh + sh * (h - 1) + 1:sh,
                     kx * dw:kx * dw + sw * (wd - 1) + 1:sw] += contrib
    y = full[:, :, ph:ph + ho, pw:pw + wo]
    if bias is not None:
        y = y + np.asarray(bias, np.float64)[None, :, None, None]
    return y


def depthwise_col2im_f32(x, w, bias=None, stride=1, pad=0, dil=1):
    """A depthwise deconvolution (group == channels == num_output) in the reference's own fp32 arithmetic and order:
    each product x w rounded to fp32 (the K = 1 gemm of backward_cpu_gemm), added by col2im into a zeroed image in
    increasing (ky, kx), then the bias added (forward_cpu_bias).  x [N, C, H, W], w [C, 1, KH, KW], bias [C] or None."""
    x, w = np.asarray(x, np.float32), np.asarray(w, np.float32)
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(pad), _pair(dil)
    n, c, h, wd = x.shape
    kh, kw = w.shape[2:]
    ho, wo = deconv_out(h, kh, sh, ph, dh), deconv_out(wd, kw, sw, pw, dw)
    y = np.zeros((n, c, ho, wo), np.float32)
    iy, ix = np.arange(h), np.arange(wd)
    for ky in range(kh):
        oy = iy * sh - ph + ky * dh
        my = (oy >= 0) & (oy < ho)
        for kx in range(kw):
            ox = ix * sw - pw + kx * dw
            mx = (ox >= 0) & (ox < wo)
            if not my.any() or not mx.any():
                continue
            prod = x[:, :, my][:, :, :, mx] * w[:, 0, ky, kx][None, :, None, None]
            # one tap reaches each output at most once: a plain fp32 add per output
            y[:, :, oy[my][:, None], ox[mx][None, :]] += prod
    if bias is not None:
        y = y + np.asarray(bias, np.float32)[None, :, None, None]
    return y


def conv_stride1(x, w, pad, dil, out_hw, group=1):
    """Stride-1 convolution in float64 with a signed pad and a given output extent: y[q] = sum_u x[q - P + u d] w[u],
    zero outside the input.  w [Cout, Cin / group, KH, KW]."""
    n, cin, h, wd = x.shape
    cout, cin_g, kh, kw = w.shape
    (ph, pw), (dh, dw), (ho, wo) = pad, dil, out_hw
    cout_g = cout // group
    y = np.zeros((n, cout, ho, wo))
    for uy in range(kh):
        for ux in range(kw):
            iy = np.arange(ho) - ph + uy * dh
            ix = np.arange(wo) - pw + ux * dw
            my, mx = (iy >= 0) & (iy < h), (ix >= 0) & (ix < wd)
            if not my.any() or not mx.any():
                continue
            yi, xi = my.nonzero()[0], mx.nonzero()[0]
            for g in range(group):
                xs = x[:, g * cin_g:(g + 1) * cin_g][:, :, iy[my]][:, :, :, ix[mx]]
                part = np.einsum("nchw,oc->nohw", xs, w[g * cout_g:(g + 1) * cout_g, :, uy, ux])
                y[:, g * cout_g:(g + 1) * cout_g, yi[:, None], xi[None, :]] += part
    return y


def phase_kernel(w, taps_h, taps_w, group=1):
    """W_r[co][ci][u_h][u_w] = w[k cin_g + ci][co - k cout_g][t_h(m_h - 1 - u_h)][t_w(m_w - 1 - u_w)]: the channel axes
    swapped per group, the taps reversed.  w [Cin, Cout / group, KH, KW] -> [Cout, Cin / group, m_h, m_w]."""
    w = np.asarray(w)
    cin, cout_g = w.shape[:2]
    cin_g = cin // group
    sub = w[:, :, taps_h[::-1]][:, :, :, taps_w[::-1]]
    return np.concatenate([sub[g * cin_g:(g + 1) * cin_g].transpose(1, 0, 2, 3) for g in range(group)], axis=0)


def phase_deconv(x, w, stride, pad, dil=1, group=1, bias=None):
    """The same deconvolution as scatter_deconv, computed as mscnn_deconv_forward does: every output phase (r_h, r_w)
    is a stride-1 convolution of x with its sub-kernel, sub-dilation and signed pad; a phase no tap reaches is the
    bias."""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(pad), _pair(dil)
    n, _, h, wd = x.shape
    cout = w.shape[1] * group
    kh, kw = w.shape[2:]
    ho, wo = deconv_out(h, kh, sh, ph, dh), deconv_out(wd, kw, sw, pw, dw)
    y = np.zeros((n, cout, ho, wo))
    for rh in range(sh):
        th, dil_h, pad_h, qh = axis_phase(kh, sh, ph, dh, ho, rh)
        for rw in range(sw):
            tw, dil_w, pad_w, qw = axis_phase(kw, sw, pw, dw, wo, rw)
            if qh == 0 or qw == 0 or not th or not tw:
                continue
            y[:, :, rh::sh, rw::sw] = conv_stride1(x, phase_kernel(w, th, tw, group), (pad_h, pad_w), (dil_h, dil_w),
                                                   (qh, qw), group)
    if bias is not None:
        y = y + np.asarray(bias, np.float64)[None, :, None, None]
    return y


def packed_elems(cin, cout, group, k, stride, pad, dil=1):
    """Elements of one plane of mscnn_pack_deconv_weights: the sub-kernels [Cout_pad][m_h][m_w][cin_g padded to 64]."""
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = _pair(k), _pair(stride), _pair(pad), _pair(dil)
    cout_pad, cin_gp = -(-cout // 64) * 64, -(-(cin // group) // 64) * 64
    return sum(len(axis_phase(kh, sh, ph, dh, 0, rh)[0]) * len(axis_phase(kw, sw, pw, dw, 0, rw)[0])
               for rh in range(sh) for rw in range(sw)) * cout_pad * cin_gp


def deconv_net(h, w, batch=2):
    """A two-convolution trunk, then: a dense k4 / s2 / p1 deconvolution with a bias (ReLU) and a grouped k2 / s2 one,
    concatenated; a convolution; a depthwise bilinear k8 / s4 / p2 deconvolution followed by a stride-4 convolution; a
    k3 / s2 / p1 deconvolution (odd output extent, ReLU) and a dilated k3 / s2 / p2 / d2 one whose odd phases no tap
    reaches, concatenated."""
    def conv(name, bottom, cout, extra, relu=True):
        s = (f'layer {{ name: "{name}" type: "Convolution" bottom: "{bottom}" top: "{name}" '
             f'convolution_param {{ num_output: {cout} {extra} }} }}\n')
        if relu:
            s += f'layer {{ name: "relu_{name}" type: "ReLU" bottom: "{name}" top: "{name}" }}\n'
        return s

    def deconv(name, bottom, cout, extra, relu=False):
        s = (f'layer {{ name: "{name}" type: "Deconvolution" bottom: "{bottom}" top: "{name}" '
             f'convolution_param {{ num_output: {cout} {extra} }} }}\n')
        if relu:
            s += f'layer {{ name: "relu_{name}" type: "ReLU" bottom: "{name}" top: "{name}" }}\n'
        return s

    def concat(name, a, b):
        return f'layer {{ name: "{name}" type: "Concat" bottom: "{a}" bottom: "{b}" top: "{name}" }}\n'

    return (f'name: "deconv"\ninput: "data"\ninput_dim: {batch} input_dim: 3 input_dim: {h} input_dim: {w}\n'
            + conv("c1", "data", 64, "kernel_size: 3 pad: 1 stride: 2")
            + conv("c2", "c1", 128, "kernel_size: 3 pad: 1")
            + deconv("d_dense", "c2", 128, "kernel_size: 4 stride: 2 pad: 1 bias_term: true", relu=True)
            + deconv("d_group", "c2", 128, "kernel_size: 2 stride: 2 group: 2 bias_term: false")
            + concat("cat_up", "d_dense", "d_group")
            + conv("c3", "cat_up", 16, "kernel_size: 3 pad: 1")
            + deconv("d_dw", "c3", 16, "kernel_size: 8 stride: 4 pad: 2 group: 16 bias_term: false")
            + conv("c4", "d_dw", 64, "kernel_size: 3 pad: 1 stride: 4")
            + deconv("d_odd", "c4", 32, "kernel_size: 3 stride: 2 pad: 1 bias_term: false", relu=True)
            + deconv("d_dil", "c4", 32, "kernel_size: 3 stride: 2 pad: 2 dilation: 2 bias_term: true")
            + concat("cat_odd", "d_odd", "d_dil"))


DECONV_BLOBS = ["c1", "c2", "d_dense", "d_group", "c3", "d_dw", "c4", "d_odd", "d_dil"]
DECONV_CONCATS = {"cat_up": ("d_dense", "d_group"), "cat_odd": ("d_odd", "d_dil")}   # copies: checked against their parts
DECONV_SIZES = [(12, 20), (9, 15)]
