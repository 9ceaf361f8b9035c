"""Image-parallel execution across the GPUs of one box (SURVEY.md section 8(e)).

Images are independent, so a global batch is split into contiguous per-rank shards with no data-path collective; the
only exchange is ONE all-gather of the final detections at the end of a step.  The reference has no multi-GPU
inference at all (its P2PSync is training-only, src/caffe/parallel.cpp:421-439).

The exchange itself lives in the C++ library (mscnn_b200/csrc/comm.cu, include/mscnn_b200.h "Multi-GPU exchange"):
`Net.detect_gather` packs this rank's final detections (header with the per-image counts + compacted rows) straight
into its slot of the gather buffer and issues one ncclAllGather on the communicator's own stream.  Python is plumbing:
`Comm` carries the 128-byte NCCL id from rank 0 to the others through torch.distributed (any backend), and
`unpack_payload` turns the gathered buffer into per-image arrays.  The gloo branch (`all_gather_payload_gloo`) moves
the same payload with torch.distributed so that the host-side logic is testable on a GPU-less machine.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from . import capi

COMM_ID_BYTES = 128


def shard_range(rank: int, per_rank: int) -> tuple[int, int]:
    """Global image indices [first, last) of a rank (weak scaling: `per_rank` images each)."""
    return rank * per_rank, (rank + 1) * per_rank


def payload_floats(batch: int, cap: int) -> int:
    """Floats per rank of the packed detection payload: int32 header [N, total, counts[N]] padded to a multiple of
    4 words, then up to batch * cap rows of [x y w h prob]; the total rounded up to a multiple of 4
    (mscnn_detect_payload_floats)."""
    return (((2 + batch + 3) & ~3) + batch * cap * 5 + 3) & ~3


def _declare(L):
    if getattr(L, "_comm_declared", False):
        return
    L.mscnn_comm_nccl_version.restype = C.c_int
    L.mscnn_comm_get_unique_id.argtypes = [C.c_void_p]
    L.mscnn_comm_init_rank.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p]
    L.mscnn_comm_init_all.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_int)]
    L.mscnn_comm_destroy.argtypes = [C.c_void_p]
    L.mscnn_comm_info.argtypes = [C.c_void_p] + [C.POINTER(C.c_int)] * 3
    L.mscnn_comm_all_gather.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.mscnn_comm_stream_wait.argtypes = [C.c_void_p, C.c_void_p]
    L.mscnn_comm_synchronize.argtypes = [C.c_void_p]
    L.mscnn_comm_gather_times.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int]
    L.mscnn_detect_payload_floats.restype = C.c_size_t
    L.mscnn_detect_payload_floats.argtypes = [C.c_int, C.c_int]
    L._comm_declared = True


class Comm:
    """One rank of the library's NCCL communicator (mscnn_comm_init_rank) on the current CUDA device.  The unique id
    is created by rank 0 and broadcast through the already initialised torch.distributed group."""

    def __init__(self, rank: int | None = None, world: int | None = None):
        self._L = capi.lib()
        _declare(self._L)
        self.rank = dist.get_rank() if rank is None else rank
        self.world = dist.get_world_size() if world is None else world
        ident = [None]
        if self.rank == 0:
            buf = C.create_string_buffer(COMM_ID_BYTES)
            capi.check(self._L.mscnn_comm_get_unique_id(buf), "comm_get_unique_id")
            ident = [bytes(buf.raw)]
        if self.world > 1:
            dist.broadcast_object_list(ident, src=0)
        self._id = C.create_string_buffer(ident[0], COMM_ID_BYTES)
        h = C.c_void_p()
        capi.check(self._L.mscnn_comm_init_rank(C.byref(h), self.world, self.rank, self._id), "comm_init_rank")
        self._h = h

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def all_gather(self, buf_all: torch.Tensor, floats_per_rank: int, stream_ptr: int) -> None:
        capi.check(self._L.mscnn_comm_all_gather(self._h, buf_all.data_ptr(), floats_per_rank, stream_ptr), "comm_all_gather")

    def stream_wait(self, stream_ptr: int) -> None:
        capi.check(self._L.mscnn_comm_stream_wait(self._h, stream_ptr), "comm_stream_wait")

    def synchronize(self) -> None:
        capi.check(self._L.mscnn_comm_synchronize(self._h), "comm_synchronize")

    def gather_times_ms(self, last: int = 64) -> list[float]:
        """Device durations of the most recent all-gathers on the communicator's stream (incl. the wait for peers)."""
        buf = (C.c_float * last)()
        n = self._L.mscnn_comm_gather_times(self._h, buf, last)
        capi.check(min(n, 0), "comm_gather_times")
        return [float(buf[i]) for i in range(n)]

    def close(self) -> None:
        if self._h:
            self._L.mscnn_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


XCHG_HANDLE_BYTES = 64


def _declare_xchg(L):
    if getattr(L, "_xchg_declared", False):
        return
    L.mscnn_xchg_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_size_t, C.c_int]
    L.mscnn_xchg_destroy.argtypes = [C.c_void_p]
    L.mscnn_xchg_ipc_handle.argtypes = [C.c_void_p, C.c_void_p]
    L.mscnn_xchg_open_peer_ipc.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.mscnn_xchg_buffer.restype = C.c_void_p
    L.mscnn_xchg_buffer.argtypes = [C.c_void_p]
    L.mscnn_xchg_wait.argtypes = [C.c_void_p, C.c_void_p]
    L.mscnn_net_detect_push.argtypes = [C.c_void_p, C.POINTER(capi.DetectCfg), C.c_void_p]
    L._xchg_declared = True


class PeerExchange:
    """One rank of the library's peer-memory exchange (mscnn_b200/csrc/xchg.cu): the post-process kernel stores this
    rank's packed detections straight into every rank's gather buffer over NVLink and raises a flag; no collective.
    The 64-byte CUDA IPC handles of the buffers travel through the initialised torch.distributed group (any backend)."""

    def __init__(self, batch: int, cap: int, rank: int | None = None, world: int | None = None, generations: int = 16):
        """generations: how many steps the ranks may drift apart (>= 2; see mscnn_xchg_create)."""
        self._L = capi.lib()
        _declare_xchg(self._L)
        self.rank = dist.get_rank() if rank is None else rank
        self.world = dist.get_world_size() if world is None else world
        self.batch, self.cap = batch, cap
        self.per = payload_floats(batch, cap)
        # Every rank walks through the same collective calls whatever happens locally, and the outcome is agreed on
        # (`self.ok`): a box where peer mapping is unavailable makes ALL ranks fall back together (bench.py: NCCL).
        self._h = None
        self.ok, self.error = True, ""
        h = C.c_void_p()
        handle = None
        try:
            capi.check(self._L.mscnn_xchg_create(C.byref(h), self.world, self.rank, self.per, generations), "xchg_create")
            self._h = h
            if self.world > 1:
                buf = C.create_string_buffer(XCHG_HANDLE_BYTES)
                capi.check(self._L.mscnn_xchg_ipc_handle(self._h, buf), "xchg_ipc_handle")
                handle = bytes(buf.raw)
        except capi.MscnnError as e:
            self.ok, self.error = False, str(e)
        if self.world > 1:
            handles = [None] * self.world
            dist.all_gather_object(handles, handle)
            if self.ok and all(hb is not None for hb in handles):
                try:
                    for p, hb in enumerate(handles):
                        if p != self.rank:
                            capi.check(self._L.mscnn_xchg_open_peer_ipc(self._h, p, C.create_string_buffer(hb, XCHG_HANDLE_BYTES)),
                                       f"xchg_open_peer_ipc({p})")
                except capi.MscnnError as e:
                    self.ok, self.error = False, str(e)
            else:
                self.ok = False
            verdicts = [None] * self.world
            dist.all_gather_object(verdicts, (self.ok, self.error))   # also the barrier: every buffer is mapped before any push
            self.ok = all(v[0] for v in verdicts)
            self.error = "; ".join(f"rank {r}: {v[1]}" for r, v in enumerate(verdicts) if v[1])
        if not self.ok:
            self.close()

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def wait(self, stream_ptr: int) -> None:
        """The stream waits (device side, no kernel) for every rank's payload of the last push."""
        capi.check(self._L.mscnn_xchg_wait(self._h, stream_ptr), "xchg_wait")

    def gathered(self) -> torch.Tensor:
        """[world * payload_floats] view of the last push's gather buffer (valid behind wait())."""
        ptr = self._L.mscnn_xchg_buffer(self._h)
        assert ptr, "nothing pushed yet"
        n = self.world * self.per
        return _cuda_view(ptr, n)

    def close(self) -> None:
        if self._h:
            self._L.mscnn_xchg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _cuda_view(ptr: int, n_floats: int) -> torch.Tensor:
    """A torch view of `n_floats` fp32 at device address `ptr` (current device), without copying."""
    class _Holder:
        pass
    h = _Holder()
    h.__cuda_array_interface__ = {"shape": (n_floats,), "typestr": "<f4", "data": (int(ptr), False), "version": 3}
    return torch.as_tensor(h, device="cuda")


def pack_payload(dets: np.ndarray, counts: np.ndarray, cap: int) -> np.ndarray:
    """Host restatement of pack_image_rows in box_output.cu (used by the CPU tests): dets [B, cap, 5], counts [B]."""
    b = len(counts)
    out = np.zeros(payload_floats(b, cap), dtype=np.float32)
    head = out.view(np.int32)
    hdr = (2 + b + 3) & ~3
    cnt = np.minimum(counts.astype(np.int64), cap)
    head[0], head[1] = b, int(cnt.sum())
    head[2:2 + b] = cnt
    rows = np.concatenate([dets[i, :cnt[i]] for i in range(b)], axis=0) if b else np.zeros((0, 5), np.float32)
    out[hdr:hdr + rows.size] = rows.reshape(-1)
    return out


def unpack_payload(payload_all: np.ndarray | torch.Tensor, world: int, batch: int, cap: int) -> list[np.ndarray]:
    """Gathered buffer [world * payload_floats] -> per global image (rank-major order = global image order) the
    [K, 5] = [x y w h prob] detections."""
    if isinstance(payload_all, torch.Tensor):
        payload_all = payload_all.detach().cpu().numpy()
    per = payload_floats(batch, cap)
    flat = np.ascontiguousarray(payload_all, dtype=np.float32).reshape(world, per)
    hdr = (2 + batch + 3) & ~3
    out = []
    for r in range(world):
        head = flat[r].view(np.int32)
        assert head[0] == batch, f"rank {r}: payload header says {head[0]} images, expected {batch}"
        counts = head[2:2 + batch]
        assert int(counts.sum()) == int(head[1])
        rows = flat[r, hdr:hdr + int(head[1]) * 5].reshape(-1, 5)
        off = 0
        for i in range(batch):
            out.append(rows[off:off + counts[i]].copy())
            off += counts[i]
    return out


def all_gather_payload_gloo(payload: torch.Tensor) -> torch.Tensor:
    """CPU / gloo stand-in for mscnn_comm_all_gather (same payload, same rank-major layout)."""
    world = dist.get_world_size()
    parts = [torch.empty_like(payload) for _ in range(world)]
    dist.all_gather(parts, payload.contiguous())
    return torch.cat(parts)
