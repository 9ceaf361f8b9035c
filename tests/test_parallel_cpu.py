"""world_size-2 gloo test of the multi-GPU plumbing on CPU tensors: sharding, the packed detection payload (header with
the per-image counts + compacted rows, the layout pack_image_rows writes) and its rank-major all-gather.  On
the GPU box the same payload is produced by the kernel and moved by ONE ncclAllGather inside libmscnn_b200.so
(mscnn_net_detect_gather; tests/test_multigpu_gpu.py, bench.py --gpus N)."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank: int, world: int, port: int, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from mscnn_b200 import parallel
    b, cap = 3, 16
    first, last = parallel.shard_range(rank, b)
    dets = np.zeros((b, cap, 5), dtype=np.float32)
    counts = np.zeros(b, dtype=np.int32)
    for i, g in enumerate(range(first, last)):      # image g has g+1 detections whose x encodes (g, k)
        counts[i] = g + 1
        for k in range(g + 1):
            dets[i, k] = [100.0 * g + k, 1, 2, 3, 0.5]
    payload = torch.from_numpy(parallel.pack_payload(dets, counts, cap))
    assert payload.numel() == parallel.payload_floats(b, cap)
    gathered = parallel.all_gather_payload_gloo(payload)
    merged = parallel.unpack_payload(gathered, world, b, cap)
    ok = len(merged) == world * b and all(
        m.shape == (g + 1, 5) and [float(v) for v in m[:, 0]] == [100.0 * g + k for k in range(g + 1)]
        for g, m in enumerate(merged))
    q.put((rank, ok))
    dist.destroy_process_group()


def test_shard_and_gather_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert res == [(0, True), (1, True)]


def test_shard_range():
    from mscnn_b200 import parallel
    assert parallel.shard_range(0, 8) == (0, 8) and parallel.shard_range(3, 8) == (24, 32)


def test_payload_roundtrip_and_size_matches_library():
    """pack -> unpack is the identity, counts above the cap are clipped, and the host-side size formula agrees with
    the library's mscnn_detect_payload_floats (no GPU needed: a pure size computation)."""
    from mscnn_b200 import capi, parallel
    L = capi.lib()
    parallel._declare(L)
    for b, cap in [(1, 5), (3, 16), (8, 2000), (6, 7)]:
        assert parallel.payload_floats(b, cap) == L.mscnn_detect_payload_floats(b, cap)
    rng = np.random.default_rng(3)
    b, cap = 4, 6
    dets = rng.standard_normal((b, cap, 5)).astype(np.float32)
    counts = np.array([0, 6, 9, 2], dtype=np.int32)          # 9 > cap: clipped to 6
    p = parallel.pack_payload(dets, counts, cap)
    out = parallel.unpack_payload(p, 1, b, cap)
    assert [len(o) for o in out] == [0, 6, 6, 2]
    for i in range(b):
        assert np.array_equal(out[i], dets[i, :min(counts[i], cap)])
