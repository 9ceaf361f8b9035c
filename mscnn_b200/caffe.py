"""pycaffe's Net and Blob over the library's net (python/caffe/pycaffe.py and _caffe.cpp of the reference), so that
Python written against a Caffe deploy net runs unchanged:

    from mscnn_b200 import caffe
    net = caffe.Net(proto, weights, caffe.TEST)
    net.blobs["data"].reshape(*x.shape)
    net.reshape()
    net.blobs["data"].data[...] = x
    net.forward()
    net.blobs["cls_pred"].data

Blob.data is the blob's host memory seen as a numpy array, fetched again on every access as pycaffe does
(Blob::mutable_cpu_data): an input written through it is uploaded by the next forward, and a weight written through
net.params[layer][i].data is packed again before the next forward.  The view is valid until the blob's next reshape.
On a net with activation reuse on (net.mscnn_net.set_activation_reuse), reading a blob whose storage a later blob took
raises MscnnError with the library's message.

The library is forward-only and runs on the GPU alone, so TRAIN, set_mode_cpu and Blob.diff are refused.  Not served:
backward, solvers, save / HDF5, set_input_arrays (MemoryData is not a registered layer type), Python layers, caffe.io,
Classifier / Detector.  The pre-processing the MS-CNN scripts do before forward is ops.Preprocess.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict
from pathlib import Path

import numpy as np

from . import capi
from . import net as mnet

TRAIN, TEST = 0, 1   # caffe.proto Phase


def set_mode_gpu() -> None:
    """The library always runs on the GPU."""


def set_mode_cpu() -> None:
    raise capi.MscnnError("set_mode_cpu: mscnn_b200 runs on the GPU only and has no CPU implementation")


def set_device(device: int) -> None:
    mnet.set_device(device)


def layer_type_list() -> list[str]:
    L = capi.lib()
    mnet._declare(L)
    buf = C.create_string_buffer(1 << 14)
    if L.mscnn_layer_type_list(buf, len(buf)) < 0:
        raise capi.MscnnError("layer_type_list failed")
    return buf.value.decode().splitlines()


def _check_file(path) -> str:
    if not Path(path).is_file():
        raise capi.MscnnError(f"Could not open file {path}")
    return str(path)


def _view(ptr: int | None, shape: tuple[int, ...], owner) -> np.ndarray:
    """float32 numpy view of `shape` at host address ptr, keeping `owner` (and so the net) alive."""
    buf = (C.c_float * int(np.prod(shape, dtype=np.int64))).from_address(ptr)
    buf._owner = owner
    return np.frombuffer(buf, dtype=np.float32).reshape(shape)


class Blob:
    """One blob of a Net, or one parameter blob of a layer (pycaffe's Blob)."""

    def __init__(self, net: "Net", name: str, param: int | None = None):
        self._net, self._name, self._param = net, name, param

    @property
    def shape(self) -> tuple[int, ...]:
        n = self._net.mscnn_net
        if self._param is not None:
            return n.param_shapes(self._name)[self._param]
        return n.blob_shape(self._name)

    def _legacy(self, axis: int) -> int:
        s = self.shape
        return s[axis] if axis < len(s) else 1

    num = property(lambda self: self._legacy(0))
    channels = property(lambda self: self._legacy(1))
    height = property(lambda self: self._legacy(2))
    width = property(lambda self: self._legacy(3))

    @property
    def count(self) -> int:
        return int(np.prod(self.shape, dtype=np.int64))

    def reshape(self, *dims: int) -> None:
        """Blob::Reshape; the net's other blobs follow at Net.reshape() or the next forward."""
        if self._param is not None:
            raise capi.MscnnError(f"parameter blob {self._param} of {self._name}: parameters keep their layer's shape")
        if len(dims) != 4:
            raise capi.MscnnError(f"reshape({', '.join(map(str, dims))}): blobs are reshaped as N x C x H x W")
        n = self._net.mscnn_net
        capi.check(n._L.mscnn_net_reshape_blob(n._h, self._name.encode(), *map(int, dims)), f"reshape({self._name})")

    @property
    def data(self) -> np.ndarray:
        n = self._net.mscnn_net
        if self._param is not None:
            ptr = n._L.mscnn_net_param_cpu_data(n._h, self._name.encode(), self._param)
            if not ptr:
                raise KeyError((self._name, self._param))
            return _view(ptr, self.shape, self)
        ptr = n._L.mscnn_net_blob_cpu_data(n._h, self._name.encode())
        if not ptr:
            msg = n._L.mscnn_net_last_error(n._h).decode()
            if msg:                                   # a released blob: say why
                raise capi.MscnnError(f"{self._name}: {msg}")
            raise KeyError(self._name)
        return _view(ptr, self.shape, self)

    @property
    def diff(self):
        raise AttributeError("diff: mscnn_b200 is forward-only and keeps no gradients")


class Layer:
    """pycaffe's Layer: its type and its parameter blobs."""

    def __init__(self, net: "Net", name: str, type_: str):
        self.type = type_
        self.blobs = [Blob(net, name, i) for i in range(len(net.mscnn_net.param_shapes(name)))]


class Net:
    """caffe.Net(proto, phase), caffe.Net(proto, weights, phase) or caffe.Net(proto, phase, weights=...).  Only TEST.

    mscnn_net is the library's net.Net behind it, for what pycaffe has no name for (activation reuse, detections,
    timing)."""

    def __init__(self, proto, *args, weights=None):
        if len(args) == 1:
            phase = args[0]
        elif len(args) == 2 and weights is None:
            weights, phase = args
        else:
            raise TypeError("Net(proto, phase), Net(proto, weights, phase) or Net(proto, phase, weights=...)")
        if phase != TEST:
            raise capi.MscnnError("Net: mscnn_b200 is forward-only; only the TEST phase is served")
        self.mscnn_net = mnet.Net(_check_file(proto))
        if weights is not None:
            self.copy_from(weights)
        n = self.mscnn_net
        self._layer_names = list(n.layer_names)
        self._blob_names = list(n.blob_names)
        self.blobs = OrderedDict((b, Blob(self, b)) for b in self._blob_names)
        self.layers = [Layer(self, l, t) for l, t in zip(n.layer_names, n.layer_types)]
        self.params = OrderedDict((l, lr.blobs) for l, lr in zip(self._layer_names, self.layers) if lr.blobs)
        self.inputs = list(n.inputs)
        self.outputs = list(n.outputs)
        self.bottom_names = self._id_names(n._L.mscnn_net_layer_bottoms)
        self.top_names = self._id_names(n._L.mscnn_net_layer_tops)

    def _id_names(self, f) -> OrderedDict:
        n, out = self.mscnn_net, OrderedDict()
        for i, l in enumerate(self._layer_names):
            ids = (C.c_int * 64)()
            k = f(n._h, i, ids, len(ids))
            if k > len(ids):
                ids = (C.c_int * k)()
                k = f(n._h, i, ids, k)
            if k < 0:
                raise capi.MscnnError(f"blob ids of layer {l} failed")
            out[l] = [self._blob_names[j] for j in ids[:k]]
        return out

    def reshape(self) -> None:
        """Net::Reshape: every blob follows the input shapes."""
        n = self.mscnn_net
        capi.check(n._L.mscnn_net_reshape(n._h), "reshape")

    def copy_from(self, path) -> None:
        self.mscnn_net.copy_from(_check_file(path))

    def share_with(self, other: "Net") -> None:
        """Net::ShareTrainedLayersWith: this net's parameters become `other`'s (one copy, one packed image each)."""
        self.mscnn_net.share_trained_layers_with(other.mscnn_net)

    def forward(self, blobs=None, start=None, end=None, **kwargs) -> dict[str, np.ndarray]:
        """pycaffe's forward: kwargs set the input blobs (all of them, each of the blob's shape), then layers start ..
        end (inclusive) run; returns copies of the outputs (of `end` when given) and of `blobs`."""
        blobs = list(blobs or [])
        outputs = ([end] if end is not None else self.outputs) + blobs
        if kwargs:
            if set(kwargs) != set(self.inputs):
                raise capi.MscnnError("Input blob arguments do not match net inputs.")
            for name, x in kwargs.items():
                if np.shape(x)[:1] != self.blobs[name].shape[:1]:
                    raise capi.MscnnError("Input is not batch sized")
                if tuple(np.shape(x)) != self.blobs[name].shape:
                    raise capi.MscnnError(f"Input {name} of shape {np.shape(x)} for a blob of shape "
                                          f"{self.blobs[name].shape}")
                self.blobs[name].data[...] = x
        self.mscnn_net.forward_only(start, end)
        return {o: self.blobs[o].data.copy() for o in dict.fromkeys(outputs)}

    def forward_all(self, blobs=None, **kwargs) -> dict[str, np.ndarray]:
        """pycaffe's forward_all: the inputs in batches of the net's batch size, the last one padded with zeros; the
        outputs concatenated along axis 0 and the padding's rows dropped."""
        all_outs = {o: [] for o in dict.fromkeys(self.outputs + list(blobs or []))}
        for batch in self._batch(kwargs):
            for o, x in self.forward(blobs=blobs, **batch).items():
                all_outs[o].extend(x.copy())
        for o in all_outs:
            all_outs[o] = np.asarray(all_outs[o])
        pad = len(next(iter(all_outs.values()))) - len(next(iter(kwargs.values())))
        if pad:
            for o in all_outs:
                all_outs[o] = all_outs[o][:-pad]
        return all_outs

    def _batch(self, blobs):
        num = len(next(iter(blobs.values())))
        batch_size = next(iter(self.blobs.values())).shape[0]
        remainder, num_batches = num % batch_size, num // batch_size
        for b in range(num_batches):
            i = b * batch_size
            yield {name: blobs[name][i:i + batch_size] for name in blobs}
        if remainder > 0:
            yield {name: np.concatenate([blobs[name][-remainder:],
                                         np.zeros((batch_size - remainder,) + blobs[name].shape[1:])])
                   for name in blobs}
