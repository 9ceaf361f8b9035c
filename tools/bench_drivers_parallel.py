"""drivers.run and widerface.run over several nets against one net, in ONE process.

KITTI car: the mscnn-8s-768 net at 768 x 2560, fp32-faithful, seeded synthetic weights, over the 64 seeded uint8 frames
of tools/bench_drivers.py (four KITTI sizes), batches of 8, host frames -> host detections.  Arms, alternated for
--rounds rounds:
  one       drivers.run(net, ...): one net, one stream, the calling thread;
  shared2   drivers.run([net, net2], ...) with net2 sharing net's weights on device 0: two host threads, two streams;
  per_gpu   drivers.run(nets, ...) with one net per visible device (only when there are two or more).
WIDER FACE: models.widerface at 32 mixed original sizes (their own net sizes, up to 1024 px), one net against two
sharing nets on device 0.

Every arm's detections are checked to equal the one-net arm's before anything is timed.  Prints one JSON object: per
arm the median and min-max of images/s over the rounds, each net's device memory (the growth of used device memory
when the net is created and runs its first forwards), and the card's name, power limit and maximum SM clock read in the
same run.

    python tools/bench_drivers_parallel.py [--rounds 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_drivers import B, KITTI, NET_H, NET_W, N_FRAMES, card  # noqa: E402

N_WIDER = 32


def used_mib(torch, device) -> float:
    torch.cuda.synchronize(device)
    free, total = torch.cuda.mem_get_info(device)
    return (total - free) / 2**20


def timed(torch, fn, devices, n_images) -> float:
    for d in devices:
        torch.cuda.synchronize(d)
    t0 = time.perf_counter()
    fn()
    for d in devices:
        torch.cuda.synchronize(d)
    return n_images / (time.perf_counter() - t0)


def stats(v):
    return {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2),
            "runs": [round(x, 2) for x in v]}


def same_fixed(a, b) -> bool:
    return len(a) == len(b) and all(x[0].tobytes() == y[0].tobytes() for x, y in zip(a, b))


def same_wider(a, b) -> bool:
    return list(a) == list(b) and all(a[k].tobytes() == b[k].tobytes() for k in a)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import numpy as np
    import torch
    from mscnn_b200 import drivers, models, net as mnet, ops, synth, widerface
    assert torch.cuda.is_available(), "bench_drivers_parallel.py needs a CUDA device"
    n_dev = torch.cuda.device_count()
    torch.cuda.set_device(0)
    mnet.set_device(0)
    mnet.set_stream(torch.cuda.current_stream().cuda_stream)
    mnet.set_precision("fp32")
    spec = drivers.KITTI_CAR
    rng = np.random.default_rng(1706)
    frames = [rng.integers(0, 256, size=(*KITTI[i % len(KITTI)], 3), dtype=np.uint8) for i in range(N_FRAMES)]
    proto = models.kitti(NET_H, NET_W, 8, False, batch=B)
    memory = {}

    # KITTI nets: each one's device memory is the growth of used memory over its creation and first run
    m0 = used_mib(torch, 0)
    one = mnet.Net(proto)
    weights = synth.make_weights(one.layers())
    one.set_params(weights)
    pre = ops.Preprocess(KITTI[0], (NET_H, NET_W))
    want = drivers.run(one, frames, spec, batch=B, pre=pre)
    memory["kitti_net_with_weights_mib"] = round(used_mib(torch, 0) - m0, 1)
    m0 = used_mib(torch, 0)
    two = mnet.Net(proto)
    two.share_trained_layers_with(one)
    pres2 = [ops.Preprocess(KITTI[0], (NET_H, NET_W)) for _ in range(2)]
    got = drivers.run([one, two], frames, spec, batch=B, pre=pres2)
    memory["kitti_sharing_net_mib"] = round(used_mib(torch, 0) - m0, 1)
    arms = {"one": (lambda: drivers.run(one, frames, spec, batch=B, pre=pre), [0]),
            "shared2": (lambda: drivers.run([one, two], frames, spec, batch=B, pre=pres2), [0])}
    identical = {"shared2": same_fixed(got, want)}
    if n_dev >= 2:
        per_gpu = [one] + drivers.make_nets(proto, weights, devices=list(range(1, n_dev)))
        pres_g = []
        for n in per_gpu:
            with torch.cuda.device(n.device):
                pres_g.append(ops.Preprocess(KITTI[0], (NET_H, NET_W)))
        got = drivers.run(per_gpu, frames, spec, batch=B, pre=pres_g)
        identical["per_gpu"] = same_fixed(got, want)
        arms["per_gpu"] = (lambda: drivers.run(per_gpu, frames, spec, batch=B, pre=pres_g), list(range(n_dev)))
    assert all(identical.values()), f"an arm gave different detections: {identical}"
    for _ in range(args.warmup):
        for fn, _devs in arms.values():
            fn()
    ips = {arm: [] for arm in arms}
    for _ in range(args.rounds):
        for arm, (fn, devs) in arms.items():
            ips[arm].append(timed(torch, fn, devs, N_FRAMES))

    # WIDER FACE: 32 frames of mixed sizes, each at its own net size, on one net and on two sharing nets
    wrng = np.random.default_rng(2017)
    wframes = []
    for k in range(N_WIDER):
        h, w = int(wrng.integers(300, 1024)), int(wrng.integers(300, 1024))
        wframes.append(wrng.integers(0, 256, size=(h, w, 3), dtype=np.uint8))
    names = [f"wider_{k}" for k in range(N_WIDER)]
    wproto = models.widerface(256, 256, batch=1)
    m0 = used_mib(torch, 0)
    w1 = mnet.Net(wproto)
    wweights = synth.make_weights(w1.layers())
    w1.set_params(wweights)
    plans1: dict = {}
    wwant = widerface.run(w1, wframes, names, plans=plans1)
    memory["wider_net_with_weights_mib"] = round(used_mib(torch, 0) - m0, 1)
    m0 = used_mib(torch, 0)
    w2 = mnet.Net(wproto)
    w2.share_trained_layers_with(w1)
    plans2 = [{}, {}]
    wgot = widerface.run([w1, w2], wframes, names, plans=plans2)
    memory["wider_sharing_net_mib"] = round(used_mib(torch, 0) - m0, 1)
    assert same_wider(wgot, wwant), "two WIDER nets gave different detections"
    warms = {"one": lambda: widerface.run(w1, wframes, names, plans=plans1),
             "shared2": lambda: widerface.run([w1, w2], wframes, names, plans=plans2)}
    for _ in range(args.warmup):
        for fn in warms.values():
            fn()
    wips = {arm: [] for arm in warms}
    for _ in range(args.rounds):
        for arm, fn in warms.items():
            wips[arm].append(timed(torch, fn, [0], N_WIDER))

    out = {"workload": f"KITTI car mscnn-8s-768 at {NET_H}x{NET_W}, fp32-faithful, {N_FRAMES} uint8 frames of four "
                       f"KITTI sizes, batches of {B}, host frames -> host detections; WIDER FACE models.widerface, "
                       f"{N_WIDER} frames of mixed sizes at their own net sizes",
           "rounds": args.rounds, **card(), "visible_gpus": n_dev, "identical_results": True,
           "kitti_images_per_s": {arm: stats(v) for arm, v in ips.items()},
           "wider_images_per_s": {arm: stats(v) for arm, v in wips.items()},
           "device_memory": memory}
    k = out["kitti_images_per_s"]
    out["kitti_shared2_over_one"] = round(k["shared2"]["median"] / k["one"]["median"], 4)
    if "per_gpu" in k:
        out["kitti_per_gpu_over_one"] = round(k["per_gpu"]["median"] / k["one"]["median"], 4)
    w = out["wider_images_per_s"]
    out["wider_shared2_over_one"] = round(w["shared2"]["median"] / w["one"]["median"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
