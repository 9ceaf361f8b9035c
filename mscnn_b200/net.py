"""Python view of the Caffe-API mirror's Net (mscnn_b200/csrc/caffe_net.cu) through the C facade
in capi_net.cu -- the counterpart of pycaffe's caffe.Net / matcaffe's caffe.Net
(/root/reference/python/caffe/pycaffe.py, matlab/+caffe/Net.m:90-109) for the forward path:

    net = Net(prototxt_path_or_text)           # deploy prototxt, TEST phase
    net.set_params(weights)                    # {layer: [blob0, blob1]} by layer name
    net.set_input("data", images)              # numpy (host) or torch.cuda tensor, NCHW fp32
    out = net.forward()                        # {'bbox_pred', 'cls_pred', 'proposals_score'}
    net.blob("conv4_3")                        # any blob, Caffe layout, as numpy

No compute happens in Python; a missing native library raises.
"""
from __future__ import annotations

import ctypes as C
import threading
from pathlib import Path

import numpy as np

from . import capi


def _declare(L):
    if getattr(L, "_net_declared", False):
        return
    L.mscnn_net_create.restype = C.c_void_p
    L.mscnn_net_create.argtypes = [C.c_char_p, C.c_int]
    L.mscnn_net_destroy.argtypes = [C.c_void_p]
    for f in ("mscnn_net_layer_name", "mscnn_net_layer_type", "mscnn_net_blob_name", "mscnn_net_input_name",
              "mscnn_net_output_name"):
        getattr(L, f).restype = C.c_char_p
        getattr(L, f).argtypes = [C.c_void_p, C.c_int]
    for f in ("mscnn_net_num_layers", "mscnn_net_num_blobs", "mscnn_net_num_inputs", "mscnn_net_num_outputs",
              "mscnn_net_reshape"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.mscnn_net_layer_param_string.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    L.mscnn_net_num_params.argtypes = [C.c_void_p, C.c_char_p]
    L.mscnn_net_param_shape.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.POINTER(C.c_int)]
    L.mscnn_net_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_long]
    L.mscnn_net_copy_trained.argtypes = [C.c_void_p, C.c_char_p]
    L.mscnn_net_share_trained_layers.argtypes = [C.c_void_p, C.c_void_p]
    L.mscnn_net_device.argtypes = [C.c_void_p]
    L.mscnn_weight_pack_count.restype = C.c_ulonglong
    L.mscnn_weight_pack_count.argtypes = []
    L.mscnn_net_get_param.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_long]
    L.mscnn_net_blob_shape.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]
    L.mscnn_net_reshape_blob.argtypes = [C.c_void_p, C.c_char_p] + [C.c_int] * 4
    L.mscnn_net_set_blob.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long]
    L.mscnn_net_set_input_images.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_void_p]
    L.mscnn_net_set_input_images_sized.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.mscnn_net_set_input_images_sized_c.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int] + [C.c_void_p] * 3
    L.mscnn_net_set_input_images_async.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_void_p]
    L.mscnn_net_set_input_images_sized_async.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int] + [C.c_void_p] * 3
    L.mscnn_net_copy_stream.restype = C.c_void_p
    L.mscnn_net_copy_stream.argtypes = [C.c_void_p]
    L.mscnn_net_set_input_geometry.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.mscnn_net_set_blob_async.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long]
    L.mscnn_net_set_blob_device.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long]
    L.mscnn_net_get_blob.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_long]
    L.mscnn_net_blob_device.restype = C.c_void_p
    L.mscnn_net_blob_device.argtypes = [C.c_void_p, C.c_char_p]
    L.mscnn_net_blob_cpu_data.restype = C.c_void_p
    L.mscnn_net_blob_cpu_data.argtypes = [C.c_void_p, C.c_char_p]
    L.mscnn_net_param_cpu_data.restype = C.c_void_p
    L.mscnn_net_param_cpu_data.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    for f in ("mscnn_net_layer_bottoms", "mscnn_net_layer_tops"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int]
    L.mscnn_layer_type_list.argtypes = [C.c_char_p, C.c_int]
    L.mscnn_net_forward.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.mscnn_net_set_layer_timing.argtypes = [C.c_void_p, C.c_int]
    L.mscnn_net_layer_times.argtypes = [C.c_void_p, C.c_void_p]
    L.mscnn_net_num_proposals.argtypes = [C.c_void_p, C.c_int]
    L.mscnn_net_detect.argtypes = [C.c_void_p, C.POINTER(capi.DetectCfg), C.c_void_p, C.c_void_p]
    L.mscnn_net_fused_producer.argtypes = [C.c_void_p, C.c_int]
    L.mscnn_net_set_graph.argtypes = [C.c_void_p, C.c_int]
    L.mscnn_net_graph_replayed.argtypes = [C.c_void_p]
    L.mscnn_net_resolve_rows.argtypes = [C.c_void_p]
    L.mscnn_net_detect_gather.restype = C.c_int
    L.mscnn_net_detect_gather.argtypes = [C.c_void_p, C.POINTER(capi.DetectCfg), C.c_void_p, C.c_void_p]
    L.mscnn_net_detect_cascade.restype = C.c_int
    L.mscnn_net_detect_cascade.argtypes = [C.c_void_p, C.POINTER(capi.DetectCfg), C.c_char_p, C.c_char_p, C.c_char_p,
                                           C.c_void_p, C.c_void_p]
    L.mscnn_net_detect_classes.restype = C.c_int
    L.mscnn_net_detect_classes.argtypes = [C.c_void_p, C.POINTER(capi.DetectCfg), C.POINTER(capi.DetectClasses),
                                           C.c_void_p, C.c_void_p]
    L.mscnn_net_detect_cascade_classes.restype = C.c_int
    L.mscnn_net_detect_cascade_classes.argtypes = [C.c_void_p, C.POINTER(capi.DetectCfg),
                                                   C.POINTER(capi.DetectClasses), C.c_char_p, C.c_char_p, C.c_char_p,
                                                   C.c_void_p, C.c_void_p]
    L.mscnn_net_detect_push_classes.restype = C.c_int
    L.mscnn_net_detect_push_classes.argtypes = [C.c_void_p, C.POINTER(capi.DetectCfg), C.POINTER(capi.DetectClasses),
                                                C.c_void_p]
    L.mscnn_net_set_activation_reuse.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.c_int]
    L.mscnn_net_activation_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.mscnn_net_activation_plan_describe.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    L.mscnn_net_activation_misses.restype = C.c_ulonglong
    L.mscnn_net_activation_misses.argtypes = [C.c_void_p]
    L.mscnn_net_last_error.restype = C.c_char_p
    L.mscnn_net_last_error.argtypes = [C.c_void_p]
    L.mscnn_set_precision.argtypes = [C.c_int]
    L.mscnn_set_stream.argtypes = [C.c_void_p]
    L.mscnn_set_device.argtypes = [C.c_int]
    L._net_declared = True


# Precision, stream and device belong to the calling host thread, as the library's Caffe context does
# (caffe_api.cu Caffe::Get): a thread that never sets them runs on the default stream in the default precision.
def set_precision(mode: str) -> None:
    """'fp32' = 3-term split-bf16 (fp32-faithful, default); 'bf16' = single bf16 term.  For this thread."""
    L = capi.lib()
    _declare(L)
    capi.check(L.mscnn_set_precision(1 if mode.lower() == "bf16" else 0), "set_precision")


def get_precision() -> str:
    """This thread's precision: 'fp32' or 'bf16'."""
    L = capi.lib()
    _declare(L)
    return "bf16" if L.mscnn_get_precision() else "fp32"


_local = threading.local()   # .stream_ptr: the stream this thread's nets run on (mscnn_set_stream); None = default


def set_stream(stream_ptr: int | None) -> None:
    """The stream the nets run on in this thread."""
    L = capi.lib()
    _declare(L)
    capi.check(L.mscnn_set_stream(stream_ptr), "set_stream")
    _local.stream_ptr = stream_ptr


def _net_stream():
    import torch
    ptr = getattr(_local, "stream_ptr", None)
    return torch.cuda.ExternalStream(ptr) if ptr else torch.cuda.default_stream()


def set_device(device: int) -> None:
    L = capi.lib()
    _declare(L)
    capi.check(L.mscnn_set_device(device), "set_device")


class Net:
    def __init__(self, prototxt: str):
        self._L = capi.lib()
        _declare(self._L)
        is_path = "\n" not in prototxt and Path(prototxt).exists()
        self._h = self._L.mscnn_net_create(str(prototxt).encode(), int(is_path))
        if not self._h:
            raise capi.MscnnError("net construction failed")
        L, h = self._L, self._h
        self.layer_names = [L.mscnn_net_layer_name(h, i).decode() for i in range(L.mscnn_net_num_layers(h))]
        self.layer_types = [L.mscnn_net_layer_type(h, i).decode() for i in range(len(self.layer_names))]
        self.blob_names = [L.mscnn_net_blob_name(h, i).decode() for i in range(L.mscnn_net_num_blobs(h))]
        self.inputs = [L.mscnn_net_input_name(h, i).decode() for i in range(L.mscnn_net_num_inputs(h))]
        self.outputs = [L.mscnn_net_output_name(h, i).decode() for i in range(L.mscnn_net_num_outputs(h))]
        self.reuse_keep: tuple[str, ...] | None = None   # set_activation_reuse: the keep set, None = reuse off

    def _check(self, rc: int, what: str) -> None:
        """capi.check, with the message of a refusal that carries one (a released blob, a refused range)."""
        if rc != capi.OK:
            msg = self._L.mscnn_net_last_error(self._h).decode()
            raise capi.MscnnError(f"{what} failed with status {rc}" + (f": {msg}" if msg else ""))

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.mscnn_net_destroy(self._h)
            self._h = None

    # ---- parameters ----------------------------------------------------------------------
    def param_shapes(self, layer: str) -> list[tuple[int, ...]]:
        n = self._L.mscnn_net_num_params(self._h, layer.encode())
        out = []
        for i in range(max(n, 0)):
            s = (C.c_int * 4)()
            nd = self._L.mscnn_net_param_shape(self._h, layer.encode(), i, s)
            out.append(tuple(s[:nd]))
        return out

    def layers(self) -> list[tuple[str, str, list[tuple[int, ...]]]]:
        return [(n, t, self.param_shapes(n)) for n, t in zip(self.layer_names, self.layer_types)]

    def layer_param_strings(self) -> list[str]:
        out = []
        for i in range(len(self.layer_names)):
            buf = C.create_string_buffer(4096)
            capi.check(self._L.mscnn_net_layer_param_string(self._h, i, buf, 4096), "layer_param_string")
            out.append(buf.value.decode())
        return out

    def set_params(self, weights: dict[str, list[np.ndarray]]) -> None:
        """Copy by layer name (Net::CopyTrainedLayersFrom semantics, net.cpp:750-785)."""
        for name, blobs in weights.items():
            if name not in self.layer_names:
                continue
            for i, b in enumerate(blobs):
                a = np.ascontiguousarray(b, dtype=np.float32)
                capi.check(self._L.mscnn_net_set_param(self._h, name.encode(), i, a.ctypes.data, a.size),
                           f"set_param({name},{i})")

    def param(self, layer: str, idx: int) -> np.ndarray:
        shp = self.param_shapes(layer)[idx]
        out = np.empty(shp, dtype=np.float32)
        capi.check(self._L.mscnn_net_get_param(self._h, layer.encode(), idx, out.ctypes.data, out.size), "get_param")
        return out

    def param_checksums(self) -> dict[str, list[float]]:
        return {n: [float(np.abs(self.param(n, i).astype(np.float64)).sum()) for i in range(len(sh))]
                for n, _, sh in self.layers() if sh}

    def copy_from(self, caffemodel: str) -> None:
        capi.check(self._L.mscnn_net_copy_trained(self._h, str(caffemodel).encode()), "copy_trained")

    def share_trained_layers_with(self, other: "Net") -> None:
        """Net::ShareTrainedLayersWith (pycaffe's share_with): every parameter blob of a layer `other` also has shares
        `other`'s storage, so a write through either net is seen by both, and both read one packed image of each
        weight (this net then allocates no weight memory).  Both nets must be on one device; the two may then run
        forwards at the same time from two host threads, each on its own stream (drivers.run over several nets).
        Raises MscnnError on a blob count or shape mismatch or different devices, sharing nothing."""
        capi.check(self._L.mscnn_net_share_trained_layers(self._h, other._h), "share_trained_layers")

    @property
    def device(self) -> int:
        """The device that was current when the net was created: where its blobs live (-1: none)."""
        return int(self._L.mscnn_net_device(self._h))

    # ---- blobs ---------------------------------------------------------------------------
    def blob_shape(self, name: str) -> tuple[int, ...]:
        s = (C.c_int * 4)()
        nd = self._L.mscnn_net_blob_shape(self._h, name.encode(), s)
        if nd < 0:
            raise KeyError(name)
        return tuple(s[:nd])

    def reshape_input(self, name: str, n: int, c: int, h: int, w: int) -> None:
        capi.check(self._L.mscnn_net_reshape_blob(self._h, name.encode(), n, c, h, w), "reshape_blob")
        capi.check(self._L.mscnn_net_reshape(self._h), "reshape")

    def set_input(self, name: str, data) -> None:
        """numpy array (host, copied H2D on the net stream) or torch CUDA tensor (D2D)."""
        shp = tuple(data.shape) + (1,) * (4 - len(data.shape))
        if self.blob_shape(name) != tuple(data.shape):
            capi.check(self._L.mscnn_net_reshape_blob(self._h, name.encode(), *shp), "reshape_blob")
        if hasattr(data, "data_ptr"):
            assert data.is_contiguous() and str(data.dtype) == "torch.float32"
            if data.is_cuda:
                rc = self._L.mscnn_net_set_blob_device(self._h, name.encode(), data.data_ptr(), data.numel())
            else:
                rc = self._L.mscnn_net_set_blob(self._h, name.encode(), data.data_ptr(), data.numel())
        else:
            a = np.ascontiguousarray(data, dtype=np.float32)
            rc = self._L.mscnn_net_set_blob(self._h, name.encode(), a.ctypes.data, a.size)
            self._keepalive = a   # the async copy reads it until the stream reaches it
        capi.check(rc, f"set_input({name})")

    def blob(self, name: str) -> np.ndarray:
        shp = self.blob_shape(name)
        out = np.empty(shp, dtype=np.float32)
        self._check(self._L.mscnn_net_get_blob(self._h, name.encode(), out.ctypes.data, out.size), f"get_blob({name})")
        return out

    def blob_device_ptr(self, name: str) -> int:
        p = self._L.mscnn_net_blob_device(self._h, name.encode())
        if not p:
            msg = self._L.mscnn_net_last_error(self._h).decode()
            if msg:                                   # a released blob: say why
                raise capi.MscnnError(f"blob_device({name}): {msg}")
            raise KeyError(name)
        return p

    # ---- activation memory -------------------------------------------------------------------
    def set_activation_reuse(self, on: bool = True, keep=()) -> None:
        """Let blobs whose lifetimes in a forward do not overlap share one device arena (Net::set_activation_reuse).
        The inputs, the outputs and the blobs named in `keep` stay readable after a forward; reading any other blob
        whose storage a later blob took raises MscnnError naming it.  on=False gives every blob its own storage back.
        Raises MscnnError for a keep name that is not a blob, changing nothing."""
        names = [str(k).encode() for k in keep]
        arr = (C.c_char_p * max(len(names), 1))(*names)
        self._check(self._L.mscnn_net_set_activation_reuse(self._h, int(bool(on)), arr, len(names)),
                    "set_activation_reuse")
        self.reuse_keep = tuple(str(k) for k in keep) if on else None

    def activation_bytes(self) -> tuple[int, int]:
        """(arena, without reuse): the bytes of the plan for the current input shapes and this thread's precision,
        and what its planned blobs take without reuse; (0, 0) with reuse off.  Host only."""
        arena, unplanned = C.c_size_t(), C.c_size_t()
        capi.check(self._L.mscnn_net_activation_bytes(self._h, C.byref(arena), C.byref(unplanned)), "activation_bytes")
        return int(arena.value), int(unplanned.value)

    def activation_plan(self) -> str:
        """The plan, one line per storage: "<blob> <bytes> <first>-<last> @<offset>" or "... input|output|kept"."""
        cap = 1 << 16
        while True:
            buf = C.create_string_buffer(cap)
            if self._L.mscnn_net_activation_plan_describe(self._h, buf, cap) == capi.OK:
                return buf.value.decode()
            cap *= 4

    def activation_misses(self) -> int:
        """Planned blobs an eager forward found without their arena storage (0 unless the plan is wrong)."""
        return int(self._L.mscnn_net_activation_misses(self._h))

    # ---- execution -----------------------------------------------------------------------
    def set_input_async(self, name: str, data) -> None:
        """Pinned host tensor / numpy array -> input blob on the copy stream, for the NEXT forward: the copy
        overlaps the rest of the forward in flight (it starts once the layers reading `name` have run)."""
        if self.blob_shape(name) != tuple(data.shape):
            raise capi.MscnnError("set_input_async does not reshape: call set_input once with this shape first")
        n = data.numel() if hasattr(data, "numel") else data.size
        assert str(data.dtype) in ("torch.float32", "float32")
        capi.check(self._L.mscnn_net_set_blob_async(self._h, name.encode(), capi.ptr(data), n), "set_blob_async")

    def set_input_images(self, name: str, pre, images) -> None:
        """uint8 host images [N][h][w][3] (numpy or pinned CPU tensor) -> device pre-processing (`pre` = an
        ops.Preprocess plan) -> the input blob; the MATLAB code before net.forward, run_mscnn_detection.m:64-69.
        A list of host uint8 [h][w][3] frames may mix original sizes: their sizes become the geometry of the next
        forward, whose detections are then rescaled and clipped per frame (run_mscnn_detection.m:64-65, 111-116).
        Gray frames ([N][h][w] / [N][h][w][1] arrays, [h][w] / [h][w][1] list entries, mixed with colour ones in a
        list) give what their repmat to three channels gives (run_cascademscnn.m:76)."""
        from . import ops
        sized = isinstance(images, (list, tuple))
        n = len(images) if sized else images.shape[0]
        shp = (n, 3, *pre.out_hw)
        if self.blob_shape(name) != shp:
            capi.check(self._L.mscnn_net_reshape_blob(self._h, name.encode(), *shp), "reshape_blob")
        if not sized and not ops.is_gray_batch(images):
            capi.check(self._L.mscnn_net_set_input_images(self._h, name.encode(), pre.handle, n, capi.ptr(images)),
                       "set_input_images")
            return
        hw, ch = ops.image_sizes_channels(images if sized else list(images))
        packed = pre.pack_host(images if sized else [images])
        gray = bool((ch == 1).any())
        if gray:
            rc = self._L.mscnn_net_set_input_images_sized_c(self._h, name.encode(), pre.handle, n, hw.ctypes.data,
                                                            ch.ctypes.data, capi.ptr(packed))
        else:
            rc = self._L.mscnn_net_set_input_images_sized(self._h, name.encode(), pre.handle, n, hw.ctypes.data,
                                                          capi.ptr(packed))
        capi.check(rc, "set_input_images_sized")
        pre.host_copy_issued(_net_stream())
        if not sized:          # an array batch records no sizes: the detect cfg's geometry applies, as for colour
            self.set_input_geometry(None)

    def set_input_images_async(self, name: str, pre, images) -> None:
        """set_input_images for the NEXT forward while the current one runs: the frames are packed into the plan's
        pinned buffer, then the H2D copy and both resize passes run on the net's copy stream once the forward in flight
        has stopped reading `name`; the next forward waits for them on the device.  The blob must already have the
        batch's shape (set_input_images reshapes, this does not).  Same frame forms and recorded sizes as
        set_input_images, so "forward k, set k + 1, detect k" pairs each batch with its own sizes."""
        from . import ops
        import torch
        sized = isinstance(images, (list, tuple))
        n = len(images) if sized else images.shape[0]
        if self.blob_shape(name) != (n, 3, *pre.out_hw):
            raise capi.MscnnError("set_input_images_async does not reshape: call set_input_images with this batch "
                                  "shape first")
        frames = images if sized else [images]
        packed = pre.pack_host(frames)
        if sized or ops.is_gray_batch(images):
            hw, ch = ops.image_sizes_channels(images if sized else list(images))
            rc = self._L.mscnn_net_set_input_images_sized_async(self._h, name.encode(), pre.handle, n, hw.ctypes.data,
                                                                ch.ctypes.data, capi.ptr(packed))
        else:
            assert tuple(images.shape[1:]) == (*pre.in_hw, 3), (images.shape, pre.in_hw)
            rc = self._L.mscnn_net_set_input_images_async(self._h, name.encode(), pre.handle, n, capi.ptr(packed))
        capi.check(rc, "set_input_images_async")
        pre.host_copy_issued(torch.cuda.ExternalStream(self._L.mscnn_net_copy_stream(self._h)))
        if not sized:
            self.set_input_geometry(None)

    def set_input_geometry(self, org_hw_list) -> None:
        """Original (h, w) of each image the NEXT forward consumes, for inputs resized by the caller and set with
        set_input*; None or [] clears them.  The detections of that forward are rescaled and clipped per image."""
        if not org_hw_list:
            capi.check(self._L.mscnn_net_set_input_geometry(self._h, 0, None), "set_input_geometry")
            return
        hw = np.ascontiguousarray(org_hw_list, dtype=np.int32).reshape(-1, 2)
        capi.check(self._L.mscnn_net_set_input_geometry(self._h, len(hw), hw.ctypes.data), "set_input_geometry")

    def forward_only(self, start: str | None = None, end: str | None = None) -> None:
        i0 = self.layer_names.index(start) if start else 0
        i1 = self.layer_names.index(end) if end else -1
        self._check(self._L.mscnn_net_forward(self._h, i0, i1), "forward")

    def forward(self, **inputs) -> dict[str, np.ndarray]:
        for k, v in inputs.items():
            self.set_input(k, v)
        self.forward_only()
        return {o: self.blob(o) for o in self.outputs}

    def num_proposals(self, image: int = -1) -> int:
        return int(self._L.mscnn_net_num_proposals(self._h, image))

    def time_layers(self) -> dict[str, float]:
        """One forward with per-layer CUDA-event timing (the `caffe time` protocol on the device)."""
        self._L.mscnn_net_set_layer_timing(self._h, 1)
        self.forward_only()
        ms = (C.c_float * len(self.layer_names))()
        self._L.mscnn_net_layer_times(self._h, ms)
        self._L.mscnn_net_set_layer_timing(self._h, 0)
        return {n: float(ms[i]) for i, n in enumerate(self.layer_names)}

    def detect(self, cfg: capi.DetectCfg, dets_dev_ptr: int, counts_dev_ptr: int) -> None:
        self._check(self._L.mscnn_net_detect(self._h, cfg, dets_dev_ptr, counts_dev_ptr), "net_detect")

    def detect_classes(self, cfg: capi.DetectCfg, classes: capi.DetectClasses, dets_dev_ptr: int,
                       counts_dev_ptr: int) -> None:
        """Final detections of several classes in one post-process (mscnn_net_detect_classes): dets
        [N][C][max_rois_per_image][5], counts [N][C], slot [n][c] = image n, class classes.cls_ids[c]."""
        self._check(self._L.mscnn_net_detect_classes(self._h, cfg, classes, dets_dev_ptr, counts_dev_ptr),
                   "net_detect_classes")

    def detect_cascade_classes(self, cfg: capi.DetectCfg, classes: capi.DetectClasses, dets_dev_ptr: int,
                               counts_dev_ptr: int, stage: str = "3rd", cls_prob: str | None = None) -> None:
        """detect_cascade for several classes: dets [N][C][max_rois_per_image][5], counts [N][C]."""
        prop = "proposals" if stage == "1st" else f"proposals_{stage}"
        self._check(self._L.mscnn_net_detect_cascade_classes(self._h, cfg, classes, prop.encode(),
                                                            (cls_prob or f"cls_prob_{stage}").encode(),
                                                            f"output_bbox_{stage}".encode(), dets_dev_ptr,
                                                            counts_dev_ptr), "net_detect_cascade_classes")

    def detect_push_classes(self, cfg: capi.DetectCfg, classes: capi.DetectClasses, xchg) -> None:
        """detect_push for several classes: the payload covers N x C slots, so `xchg` must be a
        parallel.PeerExchange made for batch * C slots (PeerExchange(batch * C, cap, ...))."""
        from . import parallel
        parallel._declare_xchg(self._L)
        self._check(self._L.mscnn_net_detect_push_classes(self._h, cfg, classes, xchg.handle), "net_detect_push_classes")

    def proposals(self, cfg: capi.DetectCfg, props_dev_ptr: int, counts_dev_ptr: int) -> None:
        """The drivers' proposal list of the last forward (mscnn_net_proposals): props float64
        [N][cfg.max_rois_per_image][5] = x y w h score in original-image coordinates, counts int32 [N]."""
        self._check(self._L.mscnn_net_proposals(self._h, cfg, props_dev_ptr, counts_dev_ptr), "net_proposals")

    def fused_producer(self, layer: str) -> str:
        """The layer that does `layer`'s work (itself unless the fusion pass folded it into another layer)."""
        i = self._L.mscnn_net_fused_producer(self._h, self.layer_names.index(layer))
        return self.layer_names[i]

    def set_graph(self, on: bool = True) -> None:
        """Replay whole forwards as one CUDA graph launch (after one eager forward; needs a non-default stream)."""
        capi.check(self._L.mscnn_net_set_graph(self._h, int(on)), "net_set_graph")

    def graph_replayed(self) -> bool:
        return bool(self._L.mscnn_net_graph_replayed(self._h))

    def detect_gather(self, cfg: capi.DetectCfg, comm, payload_all_ptr: int) -> None:
        """Final detections of this rank packed into its slot of `payload_all` + ONE all-gather on the communicator's
        stream (mscnn_net_detect_gather); `comm` is a parallel.Comm."""
        self._check(self._L.mscnn_net_detect_gather(self._h, cfg, comm.handle, payload_all_ptr), "net_detect_gather")

    def detect_push(self, cfg: capi.DetectCfg, xchg) -> None:
        """Final detections packed and pushed into every rank's gather buffer by the post-process kernel itself
        (mscnn_net_detect_push); `xchg` is a parallel.PeerExchange."""
        from . import parallel
        parallel._declare_xchg(self._L)
        self._check(self._L.mscnn_net_detect_push(self._h, cfg, xchg.handle), "net_detect_push")

    def detect_cascade(self, cfg: capi.DetectCfg, dets_dev_ptr: int, counts_dev_ptr: int, stage: str = "3rd",
                       cls_prob: str | None = None) -> None:
        """Final detections of a cascade net from one stage's blobs (run_cascademscnn.m:36-48):
        proposals[_2nd|_3rd], cls_prob_<stage> (or e.g. "cls_prob_3rd_avg"), output_bbox_<stage>."""
        prop = "proposals" if stage == "1st" else f"proposals_{stage}"
        self._check(self._L.mscnn_net_detect_cascade(self._h, cfg, prop.encode(),
                                                    (cls_prob or f"cls_prob_{stage}").encode(),
                                                    f"output_bbox_{stage}".encode(), dets_dev_ptr, counts_dev_ptr),
                   "net_detect_cascade")


def kitti_detect_cfg(net_h: int, net_w: int, max_rois: int = 2000, num_cls: int = 5, cls_id: int = 2,
                     org_hw: tuple[int, int] | None = None) -> capi.DetectCfg:
    """Post-process settings of examples/kitti_car/run_mscnn_detection.m:42-50; org_hw = size of the original
    image (`ratios = [imgH imgW] ./ [orgH orgW]`, :62-63), default = the net size (ratios = 1)."""
    cfg = capi.DetectCfg()
    cfg.num_cls, cfg.cls_id = num_cls, cls_id
    for k, v in enumerate([0.1, 0.1, 0.2, 0.2]):
        cfg.bbox_std[k] = v
        cfg.bbox_mean[k] = 0.0
    cfg.proposal_thr, cfg.nms_overlap = -10.0, 0.5
    oh, ow = org_hw if org_hw is not None else (net_h, net_w)
    cfg.ratio_h, cfg.ratio_w = net_h / oh, net_w / ow
    cfg.org_h, cfg.org_w = float(oh), float(ow)
    cfg.max_rois_per_image = max_rois
    return cfg


def kitti_ped_cyc_detect_cfg(net_h: int, net_w: int, max_rois: int = 2000,
                             org_hw: tuple[int, int] | None = None) -> tuple[capi.DetectCfg, capi.DetectClasses]:
    """Post-process settings of examples/kitti_ped_cyc/run_mscnn_detection.m:42-51 for the pedestrian / cyclist nets
    (cls_pred of 3 classes: bg, ped, cyc): the cfg and the class set cls_ids = [2 3] without a detection threshold,
    for Net.detect_classes.  Slot [n][0] holds the pedestrians, [n][1] the cyclists."""
    cfg = kitti_detect_cfg(net_h, net_w, max_rois=max_rois, num_cls=3, cls_id=2, org_hw=org_hw)
    return cfg, capi.DetectClasses.of([2, 3])


def widerface_detect_cfg(net_h: int, net_w: int, max_rois: int = 3000, org_hw: tuple[int, int] | None = None,
                         det_thr: float = 0.05) -> tuple[capi.DetectCfg, capi.DetectClasses]:
    """Post-process settings of examples/widerface/run_mscnn_detection.m:36-57 (run_cascademscnn.m:54-67): 2 classes
    (bg, face), face = class 2 with det_thr 0.05, bbox_stds [.1 .1 .2 .2], NMS overlap 0.3, proposal_thr -5.  The
    cfg and class set for Net.detect_classes / detect_cascade_classes; max_rois covers BoxOutput's max_nms_num (3000)."""
    cfg = kitti_detect_cfg(net_h, net_w, max_rois=max_rois, num_cls=2, cls_id=2, org_hw=org_hw)
    cfg.proposal_thr, cfg.nms_overlap = -5.0, 0.3
    return cfg, capi.DetectClasses.of([2], det_thr)


def image_geometry(net_hw: tuple[int, int], org_hw_list) -> np.ndarray:
    """float32 [N][4] = ratio_h, ratio_w, org_h, org_w per image (mscnn_detect_image_geometry, host only): the
    `geometry=` of ops.detect_postprocess, with the same values kitti_detect_cfg(*net_hw, org_hw=...) stores."""
    L = capi.lib()
    hw = np.ascontiguousarray(org_hw_list, dtype=np.int32).reshape(-1, 2)
    out = np.zeros((len(hw), 4), dtype=np.float32)
    capi.check(L.mscnn_detect_image_geometry(int(net_hw[0]), int(net_hw[1]), len(hw), hw.ctypes.data, out.ctypes.data),
               "detect_image_geometry")
    return out
