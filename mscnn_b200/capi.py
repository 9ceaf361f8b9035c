"""ctypes binding of the C ABI declared in include/mscnn_b200.h.

This is plumbing only: it loads the in-tree ``libmscnn_b200.so`` (built by
``python -m mscnn_b200.build``) and fails loudly when it is missing -- there is no Python or
CPU fallback for any compute entry point.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "libmscnn_b200.so"

OK = 0
ELTWISE_PROD, ELTWISE_SUM, ELTWISE_MAX = 0, 1, 2
ERR_INVALID = -1
ERR_CUDA = -2
ERR_NOMEM = -3

OUT_NHWC_BF16 = 0
OUT_NCHW_F32 = 1
OUT_NHWC_F32 = 2
POOL_MAX = 0
POOL_AVE = 1
NMS_IOU, NMS_IOMU, NMS_IOFU = 0, 1, 2
MAX_SCALES = 16

c_void_p, c_int, c_float = C.c_void_p, C.c_int, C.c_float


class MscnnError(RuntimeError):
    pass


class ConvDesc(C.Structure):
    _fields_ = [
        ("x_hi", c_void_p), ("x_lo", c_void_p),
        ("N", c_int), ("H", c_int), ("W", c_int), ("C", c_int),
        ("w_hi", c_void_p), ("w_lo", c_void_p), ("bias", c_void_p),
        ("Cout", c_int), ("Cout_pad", c_int), ("KH", c_int), ("KW", c_int),
        ("pad_h", c_int), ("pad_w", c_int),
        ("relu", c_int), ("out_mode", c_int),
        ("y_hi", c_void_p), ("y_lo", c_void_p), ("y_f32", c_void_p),
        ("pool_hi", c_void_p), ("pool_lo", c_void_p),
        ("dyn_n", c_void_p),
        # stride / dilation / groups; 0 means 1
        ("stride_h", c_int), ("stride_w", c_int), ("dil_h", c_int), ("dil_w", c_int), ("group", c_int),
    ]


class BoxOutputCfg(C.Structure):
    _fields_ = [
        ("num_scales", c_int),
        ("channels", c_int),
        ("height", c_int * MAX_SCALES), ("width", c_int * MAX_SCALES),
        ("field_w", c_float * MAX_SCALES), ("field_h", c_float * MAX_SCALES),
        ("downsample_rate", c_float * MAX_SCALES),
        ("fg_thr", c_float), ("iou_thr", c_float), ("nms_type", c_int),
        ("field_whr", c_float), ("field_xyr", c_float), ("min_size", c_float),
        ("max_nms_num", c_int), ("max_post_nms_num", c_int),
        ("do_bbox_norm", c_int),
        ("bbox_mean", c_float * 4), ("bbox_std", c_float * 4),
    ]


class DetectCfg(C.Structure):
    _fields_ = [
        ("num_cls", c_int), ("cls_id", c_int),
        ("bbox_mean", c_float * 4), ("bbox_std", c_float * 4),
        ("proposal_thr", c_float), ("nms_overlap", c_float),
        ("ratio_h", c_float), ("ratio_w", c_float), ("org_h", c_float), ("org_w", c_float),
        ("max_rois_per_image", c_int),
    ]


MAX_DETECT_CLASSES = 8


class DetectClasses(C.Structure):
    """mscnn_detect_classes: the classes of one post-process call (1-based ids, output order) and the detection
    threshold (> 0: keep prob >= det_thr before NMS; <= 0: off)."""
    _fields_ = [("num_ids", c_int), ("cls_ids", c_int * MAX_DETECT_CLASSES), ("det_thr", c_float)]

    @classmethod
    def of(cls, cls_ids, det_thr: float = -1.0) -> "DetectClasses":
        k = cls()
        ids = list(cls_ids)
        if len(ids) > MAX_DETECT_CLASSES:
            raise MscnnError(f"at most {MAX_DETECT_CLASSES} classes per post-process, got {len(ids)}")
        k.num_ids = len(ids)
        for i, v in enumerate(ids):
            k.cls_ids[i] = int(v)
        k.det_thr = float(det_thr)
        return k


class PreprocessDesc(C.Structure):
    _fields_ = [("in_h", c_int), ("in_w", c_int), ("out_h", c_int), ("out_w", c_int), ("mean", c_float * 3),
                ("swap_rb", c_int)]


_lib = None


def lib() -> C.CDLL:
    """Load (once) and return the native library; raise if it has not been built."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise MscnnError(
                f"{_LIB_PATH} is missing: run `python -m mscnn_b200.build` (nvcc, sm_90a). "
                "There is no fallback implementation.")
        _lib = C.CDLL(str(_LIB_PATH))
        _declare(_lib)
    return _lib


def _declare(L: C.CDLL) -> None:
    L.mscnn_version.restype = C.c_char_p
    L.mscnn_version.argtypes = []
    L.mscnn_sm_count.restype = c_int
    L.mscnn_kernel_launch_count.restype = C.c_ulonglong
    L.mscnn_kernel_launch_count.argtypes = []
    L.mscnn_config_reload.restype = None
    L.mscnn_config_reload.argtypes = []
    L.mscnn_conv_forward.restype = c_int
    L.mscnn_conv_forward.argtypes = [C.POINTER(ConvDesc), c_void_p]
    L.mscnn_conv_plan_describe.restype = c_int
    L.mscnn_conv_plan_describe.argtypes = [C.POINTER(ConvDesc), C.c_char_p, c_int]
    L.mscnn_conv_plan_count.restype = c_int
    L.mscnn_conv_plan_count.argtypes = []
    L.mscnn_pack_conv_weights.restype = c_int
    L.mscnn_pack_conv_weights.argtypes = [c_void_p, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]
    L.mscnn_pack_fc_weights.restype = c_int
    L.mscnn_pack_fc_weights.argtypes = [c_void_p, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]
    L.mscnn_nchw_f32_to_planes.restype = c_int
    L.mscnn_nchw_f32_to_planes.argtypes = [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]
    L.mscnn_planes_to_nchw_f32.restype = c_int
    L.mscnn_planes_to_nchw_f32.argtypes = [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]
    L.mscnn_pool_forward.restype = c_int
    L.mscnn_pool_forward.argtypes = [c_void_p] * 4 + [c_int] * 7 + [c_void_p]
    L.mscnn_pool_output_size.restype = c_int
    L.mscnn_pool_output_size.argtypes = [c_int] * 4
    L.mscnn_pool2d_forward_dyn.restype = c_int
    L.mscnn_pool2d_forward_dyn.argtypes = [c_void_p] * 4 + [c_int] * 11 + [c_void_p, c_void_p]
    L.mscnn_deconv2x_forward.restype = c_int
    L.mscnn_deconv2x_forward.argtypes = [c_void_p] * 5 + [c_int] * 5 + [c_void_p]
    L.mscnn_deconv_depthwise_forward.restype = c_int
    L.mscnn_deconv_depthwise_forward.argtypes = [c_void_p] * 6 + [c_int] * 13 + [c_void_p]
    L.mscnn_deconv_forward.restype = c_int
    L.mscnn_deconv_forward.argtypes = [C.POINTER(ConvDesc), c_void_p]
    L.mscnn_deconv_plan_describe.restype = c_int
    L.mscnn_deconv_plan_describe.argtypes = [C.POINTER(ConvDesc), C.c_char_p, c_int]
    L.mscnn_deconv_packed_elems.restype = C.c_longlong
    L.mscnn_deconv_packed_elems.argtypes = [c_int] * 12
    L.mscnn_pack_deconv_weights.restype = c_int
    L.mscnn_pack_deconv_weights.argtypes = [c_void_p, c_void_p, c_void_p] + [c_int] * 12 + [c_void_p]
    L.mscnn_box_output_workspace_bytes.restype = c_int
    L.mscnn_box_output_workspace_bytes.argtypes = [C.POINTER(BoxOutputCfg), c_int, C.POINTER(C.c_size_t)]
    L.mscnn_box_output_forward.restype = c_int
    L.mscnn_box_output_forward.argtypes = [C.POINTER(BoxOutputCfg), c_int, C.POINTER(c_void_p), c_void_p,
                                           C.c_size_t, c_void_p, c_void_p, c_void_p, c_void_p]
    L.mscnn_roi_pool_forward.restype = c_int
    L.mscnn_roi_pool_forward.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                         c_int, c_int, c_float, c_float, c_void_p, c_void_p, c_int, c_int,
                                         c_void_p]
    L.mscnn_roi_align_forward.restype = c_int
    L.mscnn_roi_align_forward.argtypes = L.mscnn_roi_pool_forward.argtypes
    # data-dependent row counts: the same arguments plus a device int count before the stream
    L.mscnn_pool_forward_dyn.restype = c_int
    L.mscnn_pool_forward_dyn.argtypes = [c_void_p] * 4 + [c_int] * 7 + [c_void_p, c_void_p]
    L.mscnn_roi_pool_multi_forward.restype = c_int
    L.mscnn_roi_pool_multi_forward.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                               c_int, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                               c_int, c_void_p]
    L.mscnn_roi_pool_multi_forward_dyn.restype = c_int
    L.mscnn_roi_pool_multi_forward_dyn.argtypes = L.mscnn_roi_pool_multi_forward.argtypes[:-1] + [c_void_p, c_void_p]
    L.mscnn_roi_align_forward_dyn.restype = c_int
    L.mscnn_roi_align_forward_dyn.argtypes = L.mscnn_roi_align_forward.argtypes[:-1] + [c_void_p, c_void_p]
    L.mscnn_pack_head_weights.restype = c_int
    L.mscnn_pack_head_weights.argtypes = [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]
    L.mscnn_head_gather.restype = c_int
    L.mscnn_head_gather.argtypes = [c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]
    L.mscnn_relu_planes.restype = c_int
    L.mscnn_relu_planes.argtypes = [c_void_p, c_void_p, C.c_size_t, c_void_p]
    L.mscnn_relu_f32.restype = c_int
    L.mscnn_relu_f32.argtypes = [c_void_p, C.c_size_t, c_void_p]
    L.mscnn_concat_planes.restype = c_int
    L.mscnn_concat_planes.argtypes = [c_void_p, c_void_p, C.c_size_t, c_int, c_int, c_int, c_void_p]
    L.mscnn_decode_bbox_forward.restype = c_int
    L.mscnn_decode_bbox_forward.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.mscnn_softmax_forward.restype = c_int
    L.mscnn_softmax_forward.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
    L.mscnn_eltwise_forward.restype = c_int
    L.mscnn_eltwise_forward.argtypes = [C.POINTER(c_void_p), c_int, c_int, c_void_p, C.c_size_t, c_void_p, c_void_p]
    L.mscnn_cascade_detect_postprocess.restype = c_int
    L.mscnn_cascade_detect_postprocess.argtypes = [C.POINTER(DetectCfg), c_int] + [c_void_p] * 5 + [C.c_size_t] + \
        [c_void_p] * 3
    L.mscnn_detect_workspace_bytes.restype = c_int
    L.mscnn_detect_workspace_bytes.argtypes = [C.POINTER(DetectCfg), c_int, C.POINTER(C.c_size_t)]
    L.mscnn_detect_postprocess.restype = c_int
    L.mscnn_detect_postprocess.argtypes = [C.POINTER(DetectCfg), c_int] + [c_void_p] * 5 + [C.c_size_t] + \
        [c_void_p] * 3
    for f in ("mscnn_detect_postprocess_sized", "mscnn_cascade_detect_postprocess_sized"):
        getattr(L, f).restype = c_int
        getattr(L, f).argtypes = [C.POINTER(DetectCfg), c_int] + [c_void_p] * 5 + [C.c_size_t] + [c_void_p] * 4
    L.mscnn_detect_postprocess_packed.restype = c_int
    L.mscnn_detect_postprocess_packed.argtypes = [C.POINTER(DetectCfg), c_int] + [c_void_p] * 5 + [C.c_size_t] + \
        [c_void_p] * 2
    L.mscnn_detect_postprocess_packed_sized.restype = c_int
    L.mscnn_detect_postprocess_packed_sized.argtypes = [C.POINTER(DetectCfg), c_int] + [c_void_p] * 5 + \
        [C.c_size_t] + [c_void_p] * 3
    L.mscnn_detect_image_geometry.restype = c_int
    L.mscnn_detect_image_geometry.argtypes = [c_int, c_int, c_int, c_void_p, c_void_p]
    L.mscnn_detect_payload_floats.restype = C.c_size_t
    L.mscnn_detect_payload_floats.argtypes = [c_int, c_int]
    L.mscnn_detect_classes_workspace_bytes.restype = c_int
    L.mscnn_detect_classes_workspace_bytes.argtypes = [C.POINTER(DetectCfg), c_int, C.POINTER(DetectClasses),
                                                       C.POINTER(C.c_size_t)]
    for f in ("mscnn_detect_postprocess_classes", "mscnn_cascade_detect_postprocess_classes"):
        getattr(L, f).restype = c_int
        getattr(L, f).argtypes = [C.POINTER(DetectCfg), C.POINTER(DetectClasses), c_int] + [c_void_p] * 5 + \
            [C.c_size_t] + [c_void_p] * 4
    L.mscnn_detect_postprocess_classes_packed.restype = c_int
    L.mscnn_detect_postprocess_classes_packed.argtypes = [C.POINTER(DetectCfg), C.POINTER(DetectClasses), c_int] + \
        [c_void_p] * 5 + [C.c_size_t] + [c_void_p] * 3
    L.mscnn_proposals_postprocess.restype = c_int
    L.mscnn_proposals_postprocess.argtypes = [C.POINTER(DetectCfg), c_int, c_void_p, c_void_p, c_int, c_int] + \
        [c_void_p] * 4
    L.mscnn_net_proposals.restype = c_int
    L.mscnn_net_proposals.argtypes = [c_void_p, C.POINTER(DetectCfg), c_void_p, c_void_p]


    L.mscnn_preprocess_create.restype = c_int
    L.mscnn_preprocess_create.argtypes = [C.POINTER(PreprocessDesc), C.POINTER(c_void_p)]
    L.mscnn_preprocess_destroy.argtypes = [c_void_p]
    L.mscnn_preprocess_get_desc.argtypes = [c_void_p, C.POINTER(PreprocessDesc)]
    L.mscnn_preprocess_forward.restype = c_int
    L.mscnn_preprocess_forward.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    L.mscnn_preprocess_forward_host.restype = c_int
    L.mscnn_preprocess_forward_host.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    for f in ("mscnn_preprocess_forward_sized", "mscnn_preprocess_forward_sized_host"):
        getattr(L, f).restype = c_int
        getattr(L, f).argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    for f in ("mscnn_preprocess_forward_sized_c", "mscnn_preprocess_forward_sized_c_host"):
        getattr(L, f).restype = c_int
        getattr(L, f).argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    L.mscnn_imresize_taps.restype = c_int
    L.mscnn_imresize_taps.argtypes = [c_int, c_int]
    L.mscnn_imresize_contributions.restype = c_int
    L.mscnn_imresize_contributions.argtypes = [c_int, c_int, c_void_p, c_void_p, c_int]
    L.mscnn_widerface_net_size.restype = c_int
    L.mscnn_widerface_net_size.argtypes = [c_int] * 5 + [C.POINTER(c_int)] * 2


    L.mscnn_kitti_write_det_file.restype = c_int
    L.mscnn_kitti_write_det_file.argtypes = [C.c_char_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int]
    L.mscnn_kitti_write_labels.restype = c_int
    L.mscnn_kitti_write_labels.argtypes = [C.c_char_p] * 5 + [C.c_double]
    L.mscnn_kitti_evaluate.restype = c_int
    L.mscnn_kitti_evaluate.argtypes = [C.c_char_p] * 3 + [c_void_p]
    L.mscnn_widerface_write_results.restype = c_int
    L.mscnn_widerface_write_results.argtypes = [C.c_char_p, c_int, C.POINTER(C.c_char_p), c_void_p, c_void_p, c_int]


    L.mscnn_conv1_tc_packed_bytes.restype = c_int
    L.mscnn_pack_conv1_tc_weights.restype = c_int
    L.mscnn_pack_conv1_tc_weights.argtypes = [c_void_p, c_void_p, c_int, c_void_p]
    L.mscnn_conv1_tc_forward.restype = c_int
    L.mscnn_conv1_tc_forward.argtypes = [c_void_p] * 5 + [c_int] * 4 + [c_void_p]


def check(rc: int, what: str = "") -> None:
    if rc != OK:
        raise MscnnError(f"{what or 'mscnn call'} failed with status {rc}")


def ptr(t) -> int | None:
    """Device/host address of a torch tensor or numpy array (None passes NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data
