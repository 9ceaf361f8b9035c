"""Cost of batching frames of different original sizes, in ONE process: the bench net (mscnn-8s-768, batch 8, fp32-
faithful, seeded weights) fed with pinned uint8 frames through Net.set_input_images, then forward, detect and the D2H
copy of the detections, for three inputs alternated over --rounds rounds:
  uniform       8 frames of 375 x 1242 as one [8][375][1242][3] array (the array entry, what bench.py times);
  uniform_list  the same 8 frames as a list (the sized entry: packing into the plan's pinned buffer + per-image
                descriptors), which separates the cost of the list form from the cost of mixed sizes;
  mixed         8 frames of four KITTI sizes (375x1242, 370x1224, 374x1238, 376x1241; the same order of pixel count),
                detections rescaled and clipped per frame.
Pre-processing alone (ops.Preprocess on the same pinned frames, H2D included) is timed with CUDA events as well.

Prints one JSON object: per arm the median and max-min spread of the per-round medians in ms, plus the card's name,
power limit and maximum SM clock read in the same run.

    python tools/bench_mixed_sizes.py [--rounds 5] [--steps 5] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

NET_H, NET_W, B = 768, 2560, 8
KITTI = [(375, 1242), (370, 1224), (374, 1238), (376, 1241)]


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, plim, smax = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax)}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None, "sm_max_mhz": None}


def stats(xs: list[float]) -> dict:
    return {"median": round(statistics.median(xs), 3), "spread": round(max(xs) - min(xs), 3),
            "runs": [round(x, 3) for x in xs]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5, help="timed steps per arm and round (the round's median is kept)")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    from mscnn_b200 import models, net as mnet, ops, synth
    assert torch.cuda.is_available(), "bench_mixed_sizes.py needs a CUDA device"
    torch.cuda.set_device(0)
    mnet.set_device(0)
    mnet.set_stream(torch.cuda.current_stream().cuda_stream)
    mnet.set_precision("fp32")
    net = mnet.Net(models.kitti(NET_H, NET_W, 8, False, batch=B))
    net.set_params(synth.make_weights(net.layers()))
    cfg = mnet.kitti_detect_cfg(NET_H, NET_W, org_hw=KITTI[0])
    cap = cfg.max_rois_per_image
    dets = torch.zeros((B, cap, 5), device="cuda")
    cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    host_dets = torch.zeros((B, cap, 5)).pin_memory()
    host_cnt = torch.zeros(B, dtype=torch.int32).pin_memory()
    rng = np.random.default_rng(1706)
    frame = lambda h, w: torch.from_numpy(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)).pin_memory()
    uniform = torch.stack([frame(*KITTI[0]) for _ in range(B)]).pin_memory()
    inputs = {"uniform": uniform, "uniform_list": [uniform[i] for i in range(B)],
              "mixed": [frame(*KITTI[i % len(KITTI)]) for i in range(B)]}
    pre = ops.Preprocess(KITTI[0], (NET_H, NET_W))
    data = torch.empty((B, 3, NET_H, NET_W), device="cuda")

    def step(images):
        net.set_input_images("data", pre, images)
        net.forward_only()
        net.detect(cfg, dets.data_ptr(), cnt.data_ptr())
        host_dets.copy_(dets, non_blocking=True)
        host_cnt.copy_(cnt, non_blocking=True)
        torch.cuda.current_stream().synchronize()

    def timed(fn, images, steps):
        ms = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(images)
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return statistics.median(ms)

    for images in inputs.values():         # warm every shape, plan entry and module of all arms
        for _ in range(args.warmup):
            step(images)
            pre(images, out=data)
    torch.cuda.synchronize()
    e2e = {arm: [] for arm in inputs}
    pre_ms = {arm: [] for arm in inputs}
    for _ in range(args.rounds):
        for arm, images in inputs.items():
            e2e[arm].append(timed(step, images, args.steps))
            pre_ms[arm].append(timed(lambda im: pre(im, out=data), images, 4 * args.steps))
    out = {"workload": "mscnn-8s-768, batch 8, fp32-faithful: set_input_images (pinned uint8) / forward / detect / D2H",
           "rounds": args.rounds, "steps": args.steps, **card(),
           "e2e_step_ms": {arm: stats(v) for arm, v in e2e.items()},
           "preprocess_ms": {arm: stats(v) for arm, v in pre_ms.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
