"""Thin torch-tensor conveniences over the C ABI (used by tests, bench.py and the Python
mirror of the Caffe Net).  torch is used for device memory and streams only; every function
here ends in exactly one C-ABI call and raises if the native library is missing.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import capi


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def reload_config() -> None:
    """Re-read the MSCNN_* environment switches (they are read once per process / per Net otherwise)."""
    capi.lib().mscnn_config_reload()


def pad64(c: int) -> int:
    return (c + 63) // 64 * 64


@dataclass
class Planes:
    """NHWC bf16 activation planes [N][H][W][Cpad]; ``lo`` is None on the plain-bf16 path."""
    hi: torch.Tensor
    lo: torch.Tensor | None
    channels: int  # logical channel count (<= Cpad)

    @property
    def shape(self):
        return tuple(self.hi.shape)

    def float(self) -> torch.Tensor:
        v = self.hi.float()
        if self.lo is not None:
            v = v + self.lo.float()
        return v[..., : self.channels]


@dataclass
class PackedWeights:
    hi: torch.Tensor          # [Cout_pad][KH][KW][Cin_pad] bf16
    lo: torch.Tensor | None
    bias: torch.Tensor        # fp32 [Cout_pad]
    cout: int
    kh: int
    kw: int


def nchw_to_planes(x: torch.Tensor, split: bool) -> Planes:
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    n, c, h, w = x.shape
    cp = pad64(c)
    hi = torch.empty((n, h, w, cp), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi) if split else None
    capi.check(capi.lib().mscnn_nchw_f32_to_planes(capi.ptr(x), capi.ptr(hi), capi.ptr(lo),
                                                   n, c, h, w, cp, _stream()), "nchw_f32_to_planes")
    return Planes(hi, lo, c)


def planes_to_nchw(p: Planes) -> torch.Tensor:
    n, h, w, cp = p.hi.shape
    y = torch.empty((n, p.channels, h, w), dtype=torch.float32, device=p.hi.device)
    capi.check(capi.lib().mscnn_planes_to_nchw_f32(capi.ptr(p.hi), capi.ptr(p.lo), capi.ptr(y),
                                                   n, p.channels, h, w, cp, _stream()),
               "planes_to_nchw_f32")
    return y


def pack_conv_weights(w: torch.Tensor, b: torch.Tensor | None, split: bool,
                      cout_pad: int | None = None, cin_pad: int | None = None) -> PackedWeights:
    """w: [Cout][Cin][KH][KW] fp32 (Caffe blob 0; [Cout][Cin / group][KH][KW] of a grouped layer packs the same way),
    b: [Cout] fp32 (blob 1) or None."""
    assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and w.dim() == 4
    cout, cin, kh, kw = w.shape
    cout_pad = cout_pad or (pad64(cout) if cout > 32 else 32)
    cin_pad = cin_pad or pad64(cin)
    hi = torch.empty((cout_pad, kh, kw, cin_pad), dtype=torch.bfloat16, device=w.device)
    lo = torch.empty_like(hi) if split else None
    capi.check(capi.lib().mscnn_pack_conv_weights(capi.ptr(w), capi.ptr(hi), capi.ptr(lo), cout, cin,
                                                  kh, kw, cout_pad, cin_pad, _stream()),
               "pack_conv_weights")
    bias = torch.zeros(cout_pad, dtype=torch.float32, device=w.device)
    if b is not None:
        bias[:cout] = b
    return PackedWeights(hi, lo, bias, cout, kh, kw)


def pack_fc_weights(w: torch.Tensor, b: torch.Tensor | None, split: bool, c: int, h: int, wd: int,
                    nout_pad: int | None = None) -> PackedWeights:
    """w: [Nout][c*h*wd] fp32 in Caffe's NCHW flattening of the bottom blob."""
    assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and w.dim() == 2
    nout = w.shape[0]
    assert w.shape[1] == c * h * wd
    nout_pad = nout_pad or (pad64(nout) if nout > 32 else 32)
    cp = pad64(c)
    hi = torch.empty((nout_pad, 1, 1, h * wd * cp), dtype=torch.bfloat16, device=w.device)
    lo = torch.empty_like(hi) if split else None
    capi.check(capi.lib().mscnn_pack_fc_weights(capi.ptr(w), capi.ptr(hi), capi.ptr(lo), nout, c, h,
                                                wd, nout_pad, cp, _stream()), "pack_fc_weights")
    bias = torch.zeros(nout_pad, dtype=torch.float32, device=w.device)
    if b is not None:
        bias[:nout] = b
    return PackedWeights(hi, lo, bias, nout, 1, 1)


def _pair(v) -> tuple[int, int]:
    return (int(v), int(v)) if isinstance(v, int) else (int(v[0]), int(v[1]))


def conv_forward(x: Planes, w: PackedWeights, pad, relu: bool, out_f32: bool = False,
                 out_split: bool | None = None, pool: str | None = None, dyn: torch.Tensor | None = None,
                 out_mode: int | None = None, out=None, stride=1, dilation=1, group: int = 1):
    """Convolution + bias (+ReLU).  Returns Planes, or an NCHW fp32 tensor when
    ``out_f32``.  An InnerProduct is the KH=KW=H=W=1 case.

    pad, stride, dilation: an int, or (h, w).  group > 1: ``w`` packed from the blob [Cout][Cin / group][KH][KW].  out_mode = capi.OUT_NHWC_F32 returns pixel-major fp32 rows
    [N][Ho][Wo][Cout_pad] (the head-tap partial sums).  dyn: a device int32 tensor of one element, the
    number of images / rows to compute (rows at or above it are left as they were).  out: a tensor or
    Planes of the returned kind to write into instead of a new one."""
    n, h, wd, c = x.hi.shape
    assert w.hi.shape[3] * group == c, (w.hi.shape, x.hi.shape, group)
    (pad_h, pad_w), (s_h, s_w), (d_h, d_w) = _pair(pad), _pair(stride), _pair(dilation)
    ho = (h + 2 * pad_h - (d_h * (w.kh - 1) + 1)) // s_h + 1
    wo = (wd + 2 * pad_w - (d_w * (w.kw - 1) + 1)) // s_w + 1
    cout_pad = w.hi.shape[0]
    if out_mode is None:
        out_mode = capi.OUT_NCHW_F32 if out_f32 else capi.OUT_NHWC_BF16
    d = capi.ConvDesc()
    d.x_hi, d.x_lo = capi.ptr(x.hi), capi.ptr(x.lo)
    d.N, d.H, d.W, d.C = n, h, wd, c
    d.w_hi, d.w_lo, d.bias = capi.ptr(w.hi), capi.ptr(w.lo), capi.ptr(w.bias)
    d.Cout, d.Cout_pad, d.KH, d.KW, d.pad_h, d.pad_w = w.cout, cout_pad, w.kh, w.kw, pad_h, pad_w
    d.relu = int(relu)
    d.stride_h, d.stride_w, d.dil_h, d.dil_w, d.group = s_h, s_w, d_h, d_w, group
    if dyn is not None:
        assert dyn.is_cuda and dyn.dtype == torch.int32 and dyn.numel() == 1
        d.dyn_n = capi.ptr(dyn)
    if out_mode in (capi.OUT_NCHW_F32, capi.OUT_NHWC_F32):
        shape = (n, w.cout, ho, wo) if out_mode == capi.OUT_NCHW_F32 else (n, ho, wo, cout_pad)
        y = torch.empty(shape, dtype=torch.float32, device=x.hi.device) if out is None else out
        assert tuple(y.shape) == shape and y.dtype == torch.float32 and y.is_contiguous()
        d.out_mode, d.y_f32 = out_mode, capi.ptr(y)
        out = y
    else:
        assert out_mode == capi.OUT_NHWC_BF16
        if out is None:
            if out_split is None:
                out_split = x.lo is not None
            y_hi = torch.empty((n, ho, wo, cout_pad), dtype=torch.bfloat16, device=x.hi.device)
            y_lo = torch.empty_like(y_hi) if out_split else None
            out = Planes(y_hi, y_lo, w.cout)
        else:
            assert not pool and out.shape == (n, ho, wo, cout_pad)
            y_hi, y_lo = out.hi, out.lo
        d.out_mode, d.y_hi, d.y_lo = capi.OUT_NHWC_BF16, capi.ptr(y_hi), capi.ptr(y_lo)
        if pool:   # "both": conv output and its fused 2x2 max pool; "only": pooled tensor alone
            p_hi = torch.empty((n, ho // 2, wo // 2, cout_pad), dtype=torch.bfloat16, device=x.hi.device)
            p_lo = torch.empty_like(p_hi) if out_split else None
            d.pool_hi, d.pool_lo = capi.ptr(p_hi), capi.ptr(p_lo)
            pooled = Planes(p_hi, p_lo, w.cout)
            if pool == "only":
                d.y_hi, d.y_lo = None, None
                out = pooled
            else:
                out = (out, pooled)
    capi.check(capi.lib().mscnn_conv_forward(d, _stream()), "conv_forward")
    return out


def pool_forward(x: Planes, kernel, stride, mode: int = capi.POOL_MAX, dyn: torch.Tensor | None = None,
                 out: Planes | None = None, pad=0) -> Planes:
    """kernel, stride, pad: an int, or (h, w); kernel = None pools each whole image (global_pooling).
    dyn: a device int32 tensor of one element, the number of images to pool (mscnn_pool_forward_dyn);
    out: planes to write into instead of new ones."""
    n, h, w, c = x.hi.shape
    if kernel is None:
        kernel = (h, w)
    if not (isinstance(kernel, int) and isinstance(stride, int) and pad == 0):
        return _pool2d_forward(x, _pair(kernel), _pair(stride), _pair(pad), mode, dyn, out)
    ho = -(-(h - kernel) // stride) + 1
    wo = -(-(w - kernel) // stride) + 1
    if out is None:
        y_hi = torch.empty((n, ho, wo, c), dtype=torch.bfloat16, device=x.hi.device)
        y_lo = torch.empty_like(y_hi) if x.lo is not None else None
        out = Planes(y_hi, y_lo, x.channels)
    assert out.shape == (n, ho, wo, c)
    args = (capi.ptr(x.hi), capi.ptr(x.lo), capi.ptr(out.hi), capi.ptr(out.lo), n, h, w, c, kernel, stride, mode)
    if dyn is None:
        capi.check(capi.lib().mscnn_pool_forward(*args, _stream()), "pool_forward")
    else:
        assert dyn.is_cuda and dyn.dtype == torch.int32 and dyn.numel() == 1
        capi.check(capi.lib().mscnn_pool_forward_dyn(*args, capi.ptr(dyn), _stream()), "pool_forward_dyn")
    return out


def _pool2d_forward(x: Planes, kernel, stride, pad, mode, dyn, out) -> Planes:
    n, h, w, c = x.hi.shape
    ho = capi.lib().mscnn_pool_output_size(h, kernel[0], stride[0], pad[0])
    wo = capi.lib().mscnn_pool_output_size(w, kernel[1], stride[1], pad[1])
    if ho <= 0 or wo <= 0:
        raise capi.MscnnError(f"pooling kernel {kernel} stride {stride} pad {pad} does not fit a {h}x{w} map")
    if out is None:
        y_hi = torch.empty((n, ho, wo, c), dtype=torch.bfloat16, device=x.hi.device)
        out = Planes(y_hi, torch.empty_like(y_hi) if x.lo is not None else None, x.channels)
    assert out.shape == (n, ho, wo, c)
    if dyn is not None:
        assert dyn.is_cuda and dyn.dtype == torch.int32 and dyn.numel() == 1
    capi.check(capi.lib().mscnn_pool2d_forward_dyn(capi.ptr(x.hi), capi.ptr(x.lo), capi.ptr(out.hi), capi.ptr(out.lo),
                                                   n, h, w, c, *kernel, *stride, *pad, mode, capi.ptr(dyn), _stream()),
               "pool2d_forward_dyn")
    return out


def deconv2x_forward(x: Planes, w: torch.Tensor) -> Planes:
    """w: fp32 [C][1][4][4] (group == channels, stride 2, pad 1, no bias)."""
    n, h, wd, c = x.hi.shape
    assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and tuple(w.shape[1:]) == (1, 4, 4)
    y_hi = torch.empty((n, 2 * h, 2 * wd, c), dtype=torch.bfloat16, device=x.hi.device)
    y_lo = torch.empty_like(y_hi) if x.lo is not None else None
    capi.check(capi.lib().mscnn_deconv2x_forward(capi.ptr(x.hi), capi.ptr(x.lo), capi.ptr(w), capi.ptr(y_hi),
                                                 capi.ptr(y_lo), n, h, wd, c, w.shape[0], _stream()),
               "deconv2x_forward")
    return Planes(y_hi, y_lo, x.channels)


def deconv_out_size(size: int, k: int, stride: int, pad: int, dilation: int = 1) -> int:
    """DeconvolutionLayer::compute_output_shape (deconv_layer.cpp:8-22)."""
    return stride * (size - 1) + dilation * (k - 1) + 1 - 2 * pad


@dataclass
class PackedDeconvWeights:
    """Weights packed by output phase for mscnn_deconv_forward (mscnn_pack_deconv_weights)."""
    hi: torch.Tensor          # [elems] bf16, the phases' sub-kernels one after another
    lo: torch.Tensor | None
    bias: torch.Tensor        # fp32 [Cout_pad]
    cin: int
    cout: int
    cout_pad: int
    kernel: tuple[int, int]
    stride: tuple[int, int]
    pad: tuple[int, int]
    dilation: tuple[int, int]
    group: int


def pack_deconv_weights(w: torch.Tensor, b: torch.Tensor | None, split: bool, stride, pad, dilation=1,
                        group: int = 1) -> PackedDeconvWeights:
    """w: [Cin][Cout / group][KH][KW] fp32 (the Deconvolution layer's blob 0), b: [Cout] fp32 (blob 1) or None.
    stride, pad, dilation: an int, or (h, w); the phase split depends on them, so they are fixed at packing."""
    assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and w.dim() == 4
    cin, cout_g, kh, kw = w.shape
    cout = cout_g * group
    cout_pad = pad64(cout)
    (s_h, s_w), (p_h, p_w), (d_h, d_w) = _pair(stride), _pair(pad), _pair(dilation)
    geom = (cin, cout, group, kh, kw, s_h, s_w, p_h, p_w, d_h, d_w, cout_pad)
    elems = capi.lib().mscnn_deconv_packed_elems(*geom)
    if elems < 0:
        raise capi.MscnnError(f"deconvolution weights {tuple(w.shape)} stride {stride} pad {pad} dilation {dilation} "
                              f"group {group}: geometry not served")
    hi = torch.empty((elems,), dtype=torch.bfloat16, device=w.device)
    lo = torch.empty_like(hi) if split else None
    capi.check(capi.lib().mscnn_pack_deconv_weights(capi.ptr(w), capi.ptr(hi), capi.ptr(lo), cin, cout, group, kh, kw,
                                                    s_h, s_w, p_h, p_w, d_h, d_w, cout_pad, _stream()),
               "pack_deconv_weights")
    bias = torch.zeros(cout_pad, dtype=torch.float32, device=w.device)
    if b is not None:
        bias[:cout] = b
    return PackedDeconvWeights(hi, lo, bias, cin, cout, cout_pad, (kh, kw), (s_h, s_w), (p_h, p_w), (d_h, d_w), group)


def deconv_desc(x: Planes, w: PackedDeconvWeights, relu: bool = False) -> capi.ConvDesc:
    """The mscnn_deconv_forward descriptor of x through w, outputs unset."""
    n, h, wd, c = x.hi.shape
    d = capi.ConvDesc()
    d.x_hi, d.x_lo = capi.ptr(x.hi), capi.ptr(x.lo)
    d.N, d.H, d.W, d.C = n, h, wd, c
    d.w_hi, d.w_lo, d.bias = capi.ptr(w.hi), capi.ptr(w.lo), capi.ptr(w.bias)
    d.Cout, d.Cout_pad, (d.KH, d.KW), (d.pad_h, d.pad_w) = w.cout, w.cout_pad, w.kernel, w.pad
    d.relu = int(relu)
    d.out_mode = capi.OUT_NHWC_BF16
    (d.stride_h, d.stride_w), (d.dil_h, d.dil_w), d.group = w.stride, w.dilation, w.group
    return d


def deconv_forward(x: Planes, w: PackedDeconvWeights, relu: bool = False, out: Planes | None = None) -> Planes:
    """Deconvolution + bias (+ReLU) of planes through weights packed by pack_deconv_weights (whose kernel, stride, pad,
    dilation and group it uses): planes [N][Ho][Wo][Cout_pad].  out: planes to write into instead of new ones."""
    n, h, wd, c = x.hi.shape
    assert c == pad64(w.cin), (x.hi.shape, w.cin)
    ho = deconv_out_size(h, w.kernel[0], w.stride[0], w.pad[0], w.dilation[0])
    wo = deconv_out_size(wd, w.kernel[1], w.stride[1], w.pad[1], w.dilation[1])
    if out is None:
        y_hi = torch.empty((n, max(ho, 0), max(wo, 0), w.cout_pad), dtype=torch.bfloat16, device=x.hi.device)
        out = Planes(y_hi, torch.empty_like(y_hi) if x.lo is not None else None, w.cout)
    assert out.shape == (n, ho, wo, w.cout_pad)
    d = deconv_desc(x, w, relu)
    d.y_hi, d.y_lo = capi.ptr(out.hi), capi.ptr(out.lo)
    capi.check(capi.lib().mscnn_deconv_forward(d, _stream()), "deconv_forward")
    return out


def deconv_depthwise_forward(x: Planes, w: torch.Tensor, b: torch.Tensor | None, stride, pad, dilation=1) -> Planes:
    """Depthwise deconvolution (group == channels == num_output): w fp32 [C][1][KH][KW] (blob 0), b fp32 [C] or None.
    kernel from w; stride, pad, dilation: an int, or (h, w)."""
    n, h, wd, c = x.hi.shape
    assert w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and w.dim() == 4 and w.shape[1] == 1
    assert b is None or (b.is_cuda and b.dtype == torch.float32 and b.is_contiguous() and b.numel() == w.shape[0])
    kh, kw = w.shape[2:]
    (s_h, s_w), (p_h, p_w), (d_h, d_w) = _pair(stride), _pair(pad), _pair(dilation)
    ho, wo = deconv_out_size(h, kh, s_h, p_h, d_h), deconv_out_size(wd, kw, s_w, p_w, d_w)
    y_hi = torch.empty((n, max(ho, 0), max(wo, 0), c), dtype=torch.bfloat16, device=x.hi.device)
    y_lo = torch.empty_like(y_hi) if x.lo is not None else None
    capi.check(capi.lib().mscnn_deconv_depthwise_forward(capi.ptr(x.hi), capi.ptr(x.lo), capi.ptr(w), capi.ptr(b),
                                                         capi.ptr(y_hi), capi.ptr(y_lo), n, h, wd, c, w.shape[0], kh,
                                                         kw, s_h, s_w, p_h, p_w, d_h, d_w, _stream()),
               "deconv_depthwise_forward")
    return Planes(y_hi, y_lo, x.channels)


def make_box_cfg(maps_shapes, field_w, field_h, rate, fg_thr, iou_thr, nms_type="IOU", field_whr=2.0,
                 field_xyr=2.0, min_size=15.0, max_nms_num=2000, max_post_nms_num=0, bbox_mean=None,
                 bbox_std=None) -> capi.BoxOutputCfg:
    """maps_shapes: [(C, H, W)] per bottom, in bottom order (BoxOutputParameter, caffe.proto:1315-1329)."""
    cfg = capi.BoxOutputCfg()
    cfg.num_scales = len(maps_shapes)
    cfg.channels = maps_shapes[0][0]
    for j, (c, h, w) in enumerate(maps_shapes):
        assert c == cfg.channels
        cfg.height[j], cfg.width[j] = h, w
        cfg.field_w[j], cfg.field_h[j], cfg.downsample_rate[j] = field_w[j], field_h[j], rate[j]
    cfg.fg_thr, cfg.iou_thr = fg_thr, iou_thr
    cfg.nms_type = {"IOU": capi.NMS_IOU, "IOMU": capi.NMS_IOMU, "IOFU": capi.NMS_IOFU}.get(nms_type, capi.NMS_IOU)
    cfg.field_whr, cfg.field_xyr, cfg.min_size = field_whr, field_xyr, min_size
    cfg.max_nms_num, cfg.max_post_nms_num = max_nms_num, max_post_nms_num
    cfg.do_bbox_norm = int(bool(bbox_mean) and bool(bbox_std))
    for k in range(4):
        cfg.bbox_mean[k] = bbox_mean[k] if cfg.do_bbox_norm else 0.0
        cfg.bbox_std[k] = bbox_std[k] if cfg.do_bbox_norm else 1.0
    return cfg


def box_output_forward(cfg: capi.BoxOutputCfg, maps: list[torch.Tensor]):
    """maps: fp32 NCHW score/delta maps.  Returns (proposals[cap,5], proposals_score[cap,6],
    num_out int32[2+N]) device tensors; rows beyond num_out[0] are undefined."""
    import ctypes as C
    n = maps[0].shape[0]
    dev = maps[0].device
    for m in maps:
        assert m.is_cuda and m.dtype == torch.float32 and m.is_contiguous() and m.shape[0] == n
    nbytes = C.c_size_t(0)
    capi.check(capi.lib().mscnn_box_output_workspace_bytes(cfg, n, C.byref(nbytes)), "box_output_workspace")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    cap = max(n * cfg.max_nms_num, 1)
    rois = torch.empty((cap, 5), dtype=torch.float32, device=dev)
    rois_score = torch.empty((cap, 6), dtype=torch.float32, device=dev)
    num_out = torch.zeros(2 + n, dtype=torch.int32, device=dev)
    ptrs = (C.c_void_p * len(maps))(*[m.data_ptr() for m in maps])
    capi.check(capi.lib().mscnn_box_output_forward(cfg, n, ptrs, capi.ptr(ws), nbytes.value, capi.ptr(rois),
                                                   capi.ptr(rois_score), capi.ptr(num_out), _stream()),
               "box_output_forward")
    return rois, rois_score, num_out


def roi_pool_forward(x: Planes, rois: torch.Tensor, num_rois: int, pooled, scale: float,
                     pad_ratio: float, out: Planes | None = None, channel_offset: int = 0,
                     out_channels: int | None = None) -> Planes:
    """ROIPooling bins [R, pooled_h, pooled_w, out_channels]; pooled: an int, or (pooled_h, pooled_w)."""
    n, h, w, c = x.hi.shape
    ph, pw = _pair(pooled)
    ctot = out_channels or c
    if out is None:
        y_hi = torch.zeros((num_rois, ph, pw, ctot), dtype=torch.bfloat16, device=x.hi.device)
        y_lo = torch.zeros_like(y_hi) if x.lo is not None else None
        out = Planes(y_hi, y_lo, ctot)
    capi.check(capi.lib().mscnn_roi_pool_forward(capi.ptr(x.hi), capi.ptr(x.lo), n, h, w, c, capi.ptr(rois),
                                                 num_rois, ph, pw, scale, pad_ratio, capi.ptr(out.hi),
                                                 capi.ptr(out.lo), ctot, channel_offset, _stream()),
               "roi_pool_forward")
    return out


def roi_pool_multi_forward(x: Planes, rois: torch.Tensor, num_rois: int, pooled, scale: float,
                           pad_ratios, channel_offsets, out: Planes | None = None, out_channels: int | None = None,
                           dyn: torch.Tensor | None = None) -> Planes:
    """Up to four pad_ratio variants of one ROI set in one launch; variant i is written at channel offset
    channel_offsets[i] of a [R, pooled_h, pooled_w, out_channels] output.  pooled: an int, or (pooled_h, pooled_w).
    dyn: device int32 ROI count."""
    import ctypes as C
    n, h, w, c = x.hi.shape
    ph, pw = _pair(pooled)
    nv = len(pad_ratios)
    assert len(channel_offsets) == nv
    ctot = out_channels or nv * c
    if out is None:
        y_hi = torch.zeros((num_rois, ph, pw, ctot), dtype=torch.bfloat16, device=x.hi.device)
        y_lo = torch.zeros_like(y_hi) if x.lo is not None else None
        out = Planes(y_hi, y_lo, ctot)
    ratios = (C.c_float * max(nv, 1))(*pad_ratios)
    offs = (C.c_int * max(nv, 1))(*channel_offsets)
    args = (capi.ptr(x.hi), capi.ptr(x.lo), n, h, w, c, capi.ptr(rois), num_rois, ph, pw, scale, nv,
            C.cast(ratios, C.c_void_p), C.cast(offs, C.c_void_p), capi.ptr(out.hi), capi.ptr(out.lo), ctot)
    if dyn is None:
        capi.check(capi.lib().mscnn_roi_pool_multi_forward(*args, _stream()), "roi_pool_multi_forward")
    else:
        assert dyn.is_cuda and dyn.dtype == torch.int32 and dyn.numel() == 1
        capi.check(capi.lib().mscnn_roi_pool_multi_forward_dyn(*args, capi.ptr(dyn), _stream()),
                   "roi_pool_multi_forward_dyn")
    return out


def roi_align_forward(x: Planes, rois: torch.Tensor, num_rois: int, pooled, scale: float,
                      pad_ratio: float, out: Planes | None = None, channel_offset: int = 0,
                      out_channels: int | None = None, dyn: torch.Tensor | None = None) -> Planes:
    """ROIAlign grid [R, pooled_h+1, pooled_w+1, C] (roi_align_layer.cpp:49-139), written at channel offset
    ``channel_offset`` of an ``out_channels``-wide output.  pooled: an int, or (pooled_h, pooled_w).
    dyn: device int32 ROI count."""
    n, h, w, c = x.hi.shape
    ph, pw = _pair(pooled)
    ctot = out_channels or c
    if out is None:
        y_hi = torch.zeros((num_rois, ph + 1, pw + 1, ctot), dtype=torch.bfloat16, device=x.hi.device)
        y_lo = torch.zeros_like(y_hi) if x.lo is not None else None
        out = Planes(y_hi, y_lo, ctot)
    args = (capi.ptr(x.hi), capi.ptr(x.lo), n, h, w, c, capi.ptr(rois), num_rois, ph, pw, scale, pad_ratio,
            capi.ptr(out.hi), capi.ptr(out.lo), ctot, channel_offset)
    if dyn is None:
        capi.check(capi.lib().mscnn_roi_align_forward(*args, _stream()), "roi_align_forward")
    else:
        assert dyn.is_cuda and dyn.dtype == torch.int32 and dyn.numel() == 1
        capi.check(capi.lib().mscnn_roi_align_forward_dyn(*args, capi.ptr(dyn), _stream()), "roi_align_forward_dyn")
    return out


def decode_bbox_forward(bbox_pred: torch.Tensor, prior: torch.Tensor, mean=None, std=None) -> torch.Tensor:
    import ctypes as C
    r = prior.shape[0]
    out = torch.empty((r, 5), dtype=torch.float32, device=prior.device)
    m = (C.c_float * 4)(*mean) if mean is not None else None
    s = (C.c_float * 4)(*std) if std is not None else None
    capi.check(capi.lib().mscnn_decode_bbox_forward(capi.ptr(bbox_pred), capi.ptr(prior), r, bbox_pred.shape[1],
                                                    C.cast(m, C.c_void_p), C.cast(s, C.c_void_p), capi.ptr(out),
                                                    _stream()), "decode_bbox_forward")
    return out


def softmax_forward(x: torch.Tensor, axis: int = 1) -> torch.Tensor:
    outer = int(np.prod(x.shape[:axis])) if axis > 0 else 1
    inner = int(np.prod(x.shape[axis + 1:])) if axis + 1 < x.dim() else 1
    y = torch.empty_like(x)
    capi.check(capi.lib().mscnn_softmax_forward(capi.ptr(x), outer, x.shape[axis], inner, capi.ptr(y), _stream()),
               "softmax_forward")
    return y


def eltwise_forward(bottoms: list[torch.Tensor], op: int, coeffs=None) -> torch.Tensor:
    import ctypes as C
    y = torch.empty_like(bottoms[0])
    ptrs = (C.c_void_p * len(bottoms))(*[b.data_ptr() for b in bottoms])
    cf = (C.c_float * len(bottoms))(*coeffs) if coeffs is not None else None
    capi.check(capi.lib().mscnn_eltwise_forward(ptrs, len(bottoms), op, C.cast(cf, C.c_void_p), y.numel(),
                                                capi.ptr(y), _stream()), "eltwise_forward")
    return y


def _detect(entry: str, cfg: capi.DetectCfg, n: int, inputs, num_out, geometry):
    """Post-process through mscnn_<entry> (geometry None) or mscnn_<entry>_sized: padded dets [n, cap, 5], counts [n]."""
    import ctypes as C
    dev = inputs[0].device
    nbytes = C.c_size_t(0)
    capi.check(capi.lib().mscnn_detect_workspace_bytes(cfg, n, C.byref(nbytes)), "detect_workspace")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    dets = torch.zeros((n, cfg.max_rois_per_image, 5), dtype=torch.float32, device=dev)
    counts = torch.zeros(n, dtype=torch.int32, device=dev)
    args = (cfg, n, *map(capi.ptr, inputs), capi.ptr(num_out), capi.ptr(ws), nbytes.value, capi.ptr(dets),
            capi.ptr(counts))
    if geometry is None:
        capi.check(getattr(capi.lib(), "mscnn_" + entry)(*args, _stream()), entry)
    else:
        g = np.ascontiguousarray(geometry, dtype=np.float32)
        assert g.shape == (n, 4), (g.shape, n)
        capi.check(getattr(capi.lib(), f"mscnn_{entry}_sized")(*args, g.ctypes.data, _stream()), entry + "_sized")
    return dets, counts


def cascade_detect_postprocess(cfg: capi.DetectCfg, n: int, proposals, cls_prob, output_bbox, num_out, geometry=None):
    """geometry: None (the cfg's ratio_* / org_*) or per-image [n][4] = ratio_h, ratio_w, org_h, org_w."""
    return _detect("cascade_detect_postprocess", cfg, n, (proposals, cls_prob, output_bbox), num_out, geometry)


def detect_postprocess(cfg: capi.DetectCfg, n: int, proposals_score, cls_pred, bbox_pred, num_out, geometry=None):
    """geometry: None (the cfg's ratio_* / org_*) or per-image [n][4] = ratio_h, ratio_w, org_h, org_w."""
    return _detect("detect_postprocess", cfg, n, (proposals_score, cls_pred, bbox_pred), num_out, geometry)


def _detect_classes(entry: str, cfg: capi.DetectCfg, classes: capi.DetectClasses, n: int, inputs, num_out, geometry,
                    packed: bool = False):
    """Post-process of several classes through mscnn_<entry>: padded dets [n, C, cap, 5] + counts [n, C], or (packed)
    the payload over n * C slots."""
    import ctypes as C
    dev = inputs[0].device
    nbytes = C.c_size_t(0)
    capi.check(capi.lib().mscnn_detect_classes_workspace_bytes(cfg, n, classes, C.byref(nbytes)),
               "detect_classes_workspace")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    g = None
    if geometry is not None:
        g = np.ascontiguousarray(geometry, dtype=np.float32)
        assert g.shape == (n, 4), (g.shape, n)
    head = (cfg, classes, n, *map(capi.ptr, inputs), capi.ptr(num_out), capi.ptr(ws), nbytes.value)
    if packed:
        payload = torch.zeros(capi.lib().mscnn_detect_payload_floats(n * classes.num_ids, cfg.max_rois_per_image),
                              dtype=torch.float32, device=dev)
        capi.check(getattr(capi.lib(), "mscnn_" + entry)(*head, capi.ptr(payload), capi.ptr(g), _stream()), entry)
        return payload
    dets = torch.zeros((n, classes.num_ids, cfg.max_rois_per_image, 5), dtype=torch.float32, device=dev)
    counts = torch.zeros((n, classes.num_ids), dtype=torch.int32, device=dev)
    capi.check(getattr(capi.lib(), "mscnn_" + entry)(*head, capi.ptr(dets), capi.ptr(counts), capi.ptr(g), _stream()),
               entry)
    return dets, counts


def detect_postprocess_classes(cfg: capi.DetectCfg, classes: capi.DetectClasses, n: int, proposals_score, cls_pred,
                               bbox_pred, num_out, geometry=None):
    """Final detections of the classes `classes.cls_ids` in one post-process: dets [n][C][cap][5], counts [n][C]
    (slot [i][c] = image i, class cls_ids[c]); geometry as in detect_postprocess."""
    return _detect_classes("detect_postprocess_classes", cfg, classes, n, (proposals_score, cls_pred, bbox_pred),
                           num_out, geometry)


def cascade_detect_postprocess_classes(cfg: capi.DetectCfg, classes: capi.DetectClasses, n: int, proposals, cls_prob,
                                       output_bbox, num_out, geometry=None):
    """The cascade post-process of several classes: dets [n][C][cap][5], counts [n][C]."""
    return _detect_classes("cascade_detect_postprocess_classes", cfg, classes, n, (proposals, cls_prob, output_bbox),
                           num_out, geometry)


def detect_postprocess_classes_packed(cfg: capi.DetectCfg, classes: capi.DetectClasses, n: int, proposals_score,
                                      cls_pred, bbox_pred, num_out, geometry=None) -> torch.Tensor:
    """detect_postprocess_classes in the exchange's packed layout over n * C slots (mscnn_detect_payload_floats)."""
    return _detect_classes("detect_postprocess_classes_packed", cfg, classes, n,
                           (proposals_score, cls_pred, bbox_pred), num_out, geometry, packed=True)


def proposals_postprocess(cfg: capi.DetectCfg, n: int, proposals_score, num_out, net_hw, org_hw=None):
    """The drivers' proposal list (mscnn_proposals_postprocess): props float64 [n, cap, 5] = x y w h score in
    original-image coordinates, counts int32 [n] (-1: more kept rows than cap = cfg.max_rois_per_image).  org_hw:
    None (cfg.org_h / org_w) or per-image [n][2] = h, w."""
    dev = proposals_score.device
    props = torch.zeros((n, cfg.max_rois_per_image, 5), dtype=torch.float64, device=dev)
    counts = torch.zeros(n, dtype=torch.int32, device=dev)
    hw = None
    if org_hw is not None:
        hw = np.ascontiguousarray(org_hw, dtype=np.int32)
        assert hw.shape == (n, 2), (hw.shape, n)
    capi.check(capi.lib().mscnn_proposals_postprocess(cfg, n, capi.ptr(proposals_score), capi.ptr(num_out),
                                                      int(net_hw[0]), int(net_hw[1]), capi.ptr(hw), capi.ptr(props),
                                                      capi.ptr(counts), _stream()), "proposals_postprocess")
    return props, counts


def conv1_tc_forward(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, relu: bool, split: bool) -> Planes:
    """conv1_1 (3 -> 64, 3x3, pad 1) as the single tensor-core kernel: x [N,3,H,W] fp32 NCHW -> planes."""
    n, c, h, wd = x.shape
    assert c == 3 and tuple(w.shape) == (64, 3, 3, 3) and x.is_contiguous() and w.is_contiguous()
    L = capi.lib()
    packed = torch.empty(L.mscnn_conv1_tc_packed_bytes(), dtype=torch.uint8, device=x.device)
    capi.check(L.mscnn_pack_conv1_tc_weights(capi.ptr(w), capi.ptr(packed), int(split), _stream()), "pack_conv1_tc")
    bias = b if b is not None else torch.zeros(64, device=x.device)
    y_hi = torch.empty((n, h, wd, 64), dtype=torch.bfloat16, device=x.device)
    y_lo = torch.empty_like(y_hi) if split else None
    capi.check(L.mscnn_conv1_tc_forward(capi.ptr(x), capi.ptr(packed), capi.ptr(bias), capi.ptr(y_hi), capi.ptr(y_lo),
                                        n, h, wd, int(relu), _stream()), "conv1_tc_forward")
    return Planes(y_hi, y_lo, 64)


# ---- pre-processing (SURVEY.md 8(f)-3) ------------------------------------------------------------
def imresize_contributions(in_len: int, out_len: int) -> tuple[np.ndarray, np.ndarray]:
    """The library's imresize tap tables for one dimension (host-only call, works without a GPU)."""
    L = capi.lib()
    taps = L.mscnn_imresize_taps(in_len, out_len)
    capi.check(min(taps, 0), "imresize_taps")
    w = np.zeros((out_len, taps), dtype=np.float64)
    idx = np.zeros((out_len, taps), dtype=np.int32)
    rc = L.mscnn_imresize_contributions(in_len, out_len, w.ctypes.data, idx.ctypes.data, taps)
    capi.check(min(rc, 0), "imresize_contributions")
    return w, idx


def widerface_net_size(org_h: int, org_w: int, img_h: int = 0, img_w: int = 0, max_size: int = 2048) -> tuple[int, int]:
    import ctypes as C
    h, w = C.c_int(), C.c_int()
    capi.check(capi.lib().mscnn_widerface_net_size(org_h, org_w, img_h, img_w, max_size, C.byref(h), C.byref(w)),
               "widerface_net_size")
    return h.value, w.value


class Preprocess:
    """imresize + BGR + mean subtraction + CHW on the device (examples/kitti_car/run_mscnn_detection.m:64-69), into
    one output size.  ``in_hw`` is the size of an array batch; a list of images may mix any sizes."""

    def __init__(self, in_hw, out_hw, mean=(104.0, 117.0, 123.0), swap_rb=True):
        import ctypes as C
        d = capi.PreprocessDesc(in_hw[0], in_hw[1], out_hw[0], out_hw[1], (C.c_float * 3)(*mean), int(swap_rb))
        h = C.c_void_p()
        capi.check(capi.lib().mscnn_preprocess_create(C.byref(d), C.byref(h)), "preprocess_create")
        self.handle, self.in_hw, self.out_hw = h, tuple(in_hw), tuple(out_hw)
        self._pinned = None    # host images of a list, packed back to back for the one H2D copy
        self._copied = None    # event behind the last H2D copy from _pinned

    def __del__(self):
        if getattr(self, "handle", None):
            capi.lib().mscnn_preprocess_destroy(self.handle)
            self.handle = None

    def __call__(self, images, out: torch.Tensor | None = None) -> torch.Tensor:
        """images: uint8 [N][h][w][3], a torch.cuda tensor, or a host numpy array / CPU tensor (H2D inside); or a
        list of uint8 [h][w][3] images of any sizes, all torch.cuda tensors or all on the host.  Gray images
        ([N][h][w] or [N][h][w][1]; [h][w] or [h][w][1] in a list, mixed with colour ones) give what their repmat to
        three channels gives (run_cascademscnn.m:76)."""
        if isinstance(images, (list, tuple)):
            return self._call_sized(images, out)
        if is_gray_batch(images):
            assert tuple(images.shape[1:3]) == self.in_hw, (images.shape, self.in_hw)
            return self._call_sized(list(images), out)
        n = images.shape[0]
        assert tuple(images.shape[1:]) == (*self.in_hw, 3) and images.dtype in (torch.uint8, np.uint8)
        if out is None:
            out = torch.empty((n, 3, *self.out_hw), dtype=torch.float32, device="cuda")
        L = capi.lib()
        if isinstance(images, torch.Tensor) and images.is_cuda:
            assert images.is_contiguous()
            capi.check(L.mscnn_preprocess_forward(self.handle, n, capi.ptr(images), capi.ptr(out), _stream()),
                       "preprocess_forward")
        else:
            capi.check(L.mscnn_preprocess_forward_host(self.handle, n, capi.ptr(images), capi.ptr(out), _stream()),
                       "preprocess_forward_host")
        return out

    def _call_sized(self, images, out):
        n = len(images)
        hw, ch = image_sizes_channels(images)
        if out is None:
            out = torch.empty((n, 3, *self.out_hw), dtype=torch.float32, device="cuda")
        L = capi.lib()
        on_device = [isinstance(im, torch.Tensor) and im.is_cuda for im in images]
        if all(on_device):
            packed = torch.cat([im.reshape(-1) for im in images])
            capi.check(L.mscnn_preprocess_forward_sized_c(self.handle, n, hw.ctypes.data, ch.ctypes.data,
                                                          capi.ptr(packed), capi.ptr(out), _stream()),
                       "preprocess_forward_sized_c")
        elif not any(on_device):
            packed = self.pack_host(images)
            capi.check(L.mscnn_preprocess_forward_sized_c_host(self.handle, n, hw.ctypes.data, ch.ctypes.data,
                                                               capi.ptr(packed), capi.ptr(out), _stream()),
                       "preprocess_forward_sized_c_host")
            self.host_copy_issued(torch.cuda.current_stream())
        else:
            raise ValueError("a list of images must be all on the device or all on the host")
        return out

    def pack_host(self, images) -> torch.Tensor:
        """Host images back to back in one pinned buffer owned by the plan, so that their H2D copy is asynchronous.
        The buffer is refilled only once the copy issued from it last time has run (`host_copy_issued`)."""
        total = sum(int(np.prod(im.shape)) for im in images)
        if self._copied is not None:
            self._copied.synchronize()
        if self._pinned is None or self._pinned.numel() < total:
            self._pinned = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        off = 0
        for im in images:
            t = torch.as_tensor(im).reshape(-1)
            self._pinned[off:off + t.numel()].copy_(t)
            off += t.numel()
        return self._pinned

    def host_copy_issued(self, stream: torch.cuda.Stream) -> None:
        """Mark the H2D copy from the packed buffer, just issued on `stream`."""
        self._copied = torch.cuda.Event()
        self._copied.record(stream)


def image_sizes(images) -> np.ndarray:
    """int32 [N][2] = h, w of a list of uint8 [h][w][3] images (or gray [h][w] / [h][w][1] ones)."""
    return image_sizes_channels(images)[0]


def image_sizes_channels(images) -> tuple[np.ndarray, np.ndarray]:
    """int32 [N][2] = h, w and int32 [N] = channels (3, or 1 for a gray [h][w] / [h][w][1] image) of a list of uint8
    images; any other shape is refused."""
    assert len(images) >= 1
    for im in images:
        shp = tuple(im.shape)
        assert (len(shp) == 2 or (len(shp) == 3 and shp[2] in (1, 3))) and im.dtype in (torch.uint8, np.uint8), \
            (shp, im.dtype)
    hw = np.ascontiguousarray([im.shape[:2] for im in images], dtype=np.int32)
    ch = np.ascontiguousarray([im.shape[2] if len(im.shape) == 3 else 1 for im in images], dtype=np.int32)
    return hw, ch


def is_gray_batch(images) -> bool:
    """True for a uint8 batch array of gray images, [N][h][w] or [N][h][w][1]."""
    return len(images.shape) == 3 or (len(images.shape) == 4 and images.shape[3] == 1)
