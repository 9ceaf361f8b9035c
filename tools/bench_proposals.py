"""Cost of the drivers' proposal list (Net.proposals, drivers.run(..., proposals=True)).

Two numbers, with the card's name and power limit read in the same process:
  * the proposal stage alone on the BoxOutput rows of a batch of 8 KITTI frames (375x1242) at 768x2560: CUDA events
    around each launch, the median (and quartiles) over --launches launches after a warm-up;
  * drivers.run with KITTI_CAR's settings at 768x2560, batch 8, in images/s with proposals off and on, the two arms
    alternated over --rounds rounds, each round one run over --frames frames, after one warm-up run of each arm.
The net is the shipped kitti_car/mscnn-8s-768-trainval deploy file with synthetic weights (tests/golden/deploy.tar.xz),
fp32-faithful.  Prints one JSON line.

    python tools/bench_proposals.py [--launches 500] [--rounds 5] [--frames 32]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

NET_HW = (768, 2560)
ORG = (375, 1242)


def deploy(rel, n, h, w):
    """A shipped deploy net (tests/golden/deploy.tar.xz) with its input set to n x 3 x h x w."""
    import re
    import tarfile
    with tarfile.open(Path(__file__).resolve().parent.parent / "tests" / "golden" / "deploy.tar.xz") as t:
        text = t.extractfile(f"deploy/{rel}/mscnn_deploy.prototxt").read().decode()
    return re.sub(r"input_dim: 1\s+input_dim: 3\s+input_dim: \d+\s+input_dim: \d+",
                  f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frames(k, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(k):
        im = rng.integers(0, 256, size=(*ORG, 3), dtype=np.uint8)
        im[: ORG[0] // 3, : ORG[1] // 4] = 255
        out.append(im)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=32)
    args = ap.parse_args()
    import torch
    from mscnn_b200 import drivers, net as mnet, ops, synth
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    mnet.set_precision("fp32")
    spec = drivers.KITTI_CAR
    net = mnet.Net(deploy("kitti_car/mscnn-8s-768-trainval", 8, *NET_HW))
    net.set_params(synth.make_weights(net.layers()))
    rec = {"card": card(), "net": "kitti_car/mscnn-8s-768-trainval (synthetic weights)", "net_hw": list(NET_HW),
           "batch": 8, "precision": "fp32"}

    # the proposal stage alone
    batch = frames(8)
    net.set_input_images("data", ops.Preprocess(ORG, NET_HW), batch)
    net.forward_only()
    cfg, _ = spec.detect_cfg(NET_HW)
    props = torch.empty((8, cfg.max_rois_per_image, 5), dtype=torch.float64, device="cuda")
    counts = torch.empty(8, dtype=torch.int32, device="cuda")
    for _ in range(20):
        net.proposals(cfg, props.data_ptr(), counts.data_ptr())
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.launches)]
    for a, b in ev:
        a.record()
        net.proposals(cfg, props.data_ptr(), counts.data_ptr())
        b.record()
    torch.cuda.synchronize()
    us = np.array([a.elapsed_time(b) * 1e3 for a, b in ev])
    rec["proposal_stage_us"] = {"median": float(np.median(us)), "p25": float(np.percentile(us, 25)),
                                "p75": float(np.percentile(us, 75)), "launches": args.launches}
    rec["rows_in"] = int(net.num_proposals())
    rec["rows_kept"] = int(counts.sum().item())
    del net

    # drivers.run with and without the proposal list, arms alternated
    run_net = mnet.Net(deploy("kitti_car/mscnn-8s-768-trainval", 1, *NET_HW))
    run_net.set_params(synth.make_weights(run_net.layers()))
    fr = frames(args.frames, seed=1)
    pre = ops.Preprocess(ORG, NET_HW)
    rates = {"off": [], "on": []}
    for r in range(args.rounds + 1):
        for arm in ("off", "on") if r % 2 == 0 else ("on", "off"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            drivers.run(run_net, fr, spec, batch=8, pre=pre, proposals=(arm == "on"))
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if r > 0:                                     # round 0 warms both arms up
                rates[arm].append(len(fr) / dt)
    for arm, v in rates.items():
        rec[f"drivers_run_images_per_s_proposals_{arm}"] = {"median": float(np.median(v)), "min": float(min(v)),
                                                            "max": float(max(v)), "rounds": len(v)}
    rec["frames"] = args.frames
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
