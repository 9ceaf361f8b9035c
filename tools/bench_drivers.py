"""drivers.run against the synchronous driver loop, in ONE process: the KITTI car net (mscnn-8s-768, 768 x 2560, fp32-
faithful, seeded synthetic weights) over 64 seeded uint8 host frames of the four KITTI sizes, batches of 8, from host
frames to the kept detections on the host.  Two arms, alternated for --rounds rounds:
  sync  per batch: Net.set_input_images (pack, H2D, both resize passes), forward, detect_classes, readback; the next
        batch starts only then;
  run   drivers.run(net, frames, drivers.KITTI_CAR): the same calls, but batch k + 1 is pre-processed on the net's copy
        stream (Net.set_input_images_async) while batch k's forward runs.
Both arms' detections are checked to be identical before anything is timed.

Prints one JSON object: per arm the median and min-max of images/s over the rounds, plus the card's name, power limit
and maximum SM clock read in the same run.

    python tools/bench_drivers.py [--rounds 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

NET_H, NET_W, B, N_FRAMES = 768, 2560, 8, 64
KITTI = [(375, 1242), (370, 1224), (374, 1238), (376, 1241)]


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, plim, smax = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax)}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None, "sm_max_mhz": None}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import numpy as np
    import torch
    from mscnn_b200 import drivers, models, net as mnet, ops, synth
    assert torch.cuda.is_available(), "bench_drivers.py needs a CUDA device"
    torch.cuda.set_device(0)
    mnet.set_device(0)
    mnet.set_stream(torch.cuda.current_stream().cuda_stream)
    mnet.set_precision("fp32")
    spec = drivers.KITTI_CAR
    net = mnet.Net(models.kitti(NET_H, NET_W, 8, False, batch=B))
    net.set_params(synth.make_weights(net.layers()))
    rng = np.random.default_rng(1706)
    frames = [rng.integers(0, 256, size=(*KITTI[i % len(KITTI)], 3), dtype=np.uint8) for i in range(N_FRAMES)]
    pre = ops.Preprocess(KITTI[0], (NET_H, NET_W))
    cfg, classes = spec.detect_cfg()
    cap = cfg.max_rois_per_image

    def sync_loop():
        out = []
        for k in range(0, N_FRAMES, B):
            net.set_input_images("data", pre, frames[k:k + B])
            net.forward_only()
            dets = torch.empty((B, 1, cap, 5), device="cuda")
            counts = torch.empty((B, 1), dtype=torch.int32, device="cuda")
            net.detect_classes(cfg, classes, dets.data_ptr(), counts.data_ptr())
            cnt = counts.cpu().numpy()
            d = dets[:, :, :int(cnt.max())].cpu().numpy()
            out += [[d[j, 0, :cnt[j, 0]].copy()] for j in range(B)]
        return out

    def pipelined():
        return drivers.run(net, frames, spec, batch=B, pre=pre)

    arms = {"sync": sync_loop, "run": pipelined}
    first = {arm: fn() for arm, fn in arms.items()}
    same = all(a[0].tobytes() == b[0].tobytes() for a, b in zip(first["sync"], first["run"]))
    assert same, "the two arms gave different detections"
    kept = sum(len(r[0]) for r in first["run"])
    for _ in range(args.warmup):
        for fn in arms.values():
            fn()
    ips = {arm: [] for arm in arms}
    for _ in range(args.rounds):
        for arm, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ips[arm].append(N_FRAMES / (time.perf_counter() - t0))
    out = {"workload": f"KITTI car mscnn-8s-768 at {NET_H}x{NET_W}, fp32-faithful, {N_FRAMES} uint8 frames of four "
                       f"KITTI sizes, batches of {B}, host frames -> host detections",
           "rounds": args.rounds, **card(), "identical_results": same, "kept_detections": kept,
           "images_per_s": {arm: {"median": round(statistics.median(v), 2), "min": round(min(v), 2),
                                  "max": round(max(v), 2), "runs": [round(x, 2) for x in v]} for arm, v in ips.items()}}
    out["run_over_sync"] = round(out["images_per_s"]["run"]["median"] / out["images_per_s"]["sync"]["median"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
