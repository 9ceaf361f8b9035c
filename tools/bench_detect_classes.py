"""Final detections of the KITTI pedestrian / cyclist net: two single-class post-processes (what a caller of
mscnn_net_detect needs for cls_ids = [2 3], examples/kitti_ped_cyc/run_mscnn_detection.m:48,93-121) against one
mscnn_net_detect_classes call over both classes.  Not the bench line (bench.py measures the car net's forward).

    python tools/bench_detect_classes.py [--batch 8] [--rounds 30] [--reps 20]

The post-process inputs come from one forward of the shipped kitti_ped_cyc/mscnn-8s-768-trainval deploy net
(tests/golden/deploy.tar.xz) at batch x 3 x 768 x 2560 with synthetic weights and images (mscnn_b200/synth.py).  Each
round times `reps` back-to-back calls of each arm with CUDA events, the arms alternating inside the round; the result
is the median and spread over rounds of the per-call time, with the card's name and power limit read in the same run.
Both arms' outputs are compared bit for bit before timing.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import re
import subprocess
import sys
import tarfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def pedcyc_deploy(n: int, h: int, w: int) -> str:
    with tarfile.open(ROOT / "tests" / "golden" / "deploy.tar.xz") as t:
        text = t.extractfile("deploy/kitti_ped_cyc/mscnn-8s-768-trainval/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: 768\s+input_dim: 2560",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def card() -> dict:
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.split(",")][:2]
    except (OSError, ValueError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--height", type=int, default=768)
    ap.add_argument("--width", type=int, default=2560)
    args = ap.parse_args()
    import numpy as np
    import torch
    from mscnn_b200 import capi, net as mnet, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_detect_classes needs a CUDA device")

    B, H, W = args.batch, args.height, args.width
    torch.cuda.set_device(0)
    mnet.set_device(0)
    mnet.set_stream(torch.cuda.current_stream().cuda_stream)
    mnet.set_precision("fp32")
    net = mnet.Net(pedcyc_deploy(B, H, W))
    net.set_params(synth.make_weights(net.layers()))
    net.forward(data=synth.make_images(B, H, W))
    cfg, k = mnet.kitti_ped_cyc_detect_cfg(H, W)
    ids = list(k.cls_ids[:k.num_ids])
    C, cap, dev = len(ids), cfg.max_rois_per_image, torch.device("cuda", 0)
    one = [(torch.zeros((B, cap, 5), device=dev), torch.zeros(B, dtype=torch.int32, device=dev)) for _ in ids]
    both = (torch.zeros((B, C, cap, 5), device=dev), torch.zeros((B, C), dtype=torch.int32, device=dev))

    def singles():
        for (d, c), cid in zip(one, ids):
            cfg.cls_id = cid
            net.detect(cfg, d.data_ptr(), c.data_ptr())

    def classes():
        net.detect_classes(cfg, k, both[0].data_ptr(), both[1].data_ptr())

    singles()
    classes()
    torch.cuda.synchronize()
    for c in range(C):
        assert torch.equal(both[1][:, c], one[c][1]) and torch.equal(both[0][:, c].view(torch.int32),
                                                                     one[c][0].view(torch.int32)), c
    L = capi.lib()

    def launches(fn):
        n0 = L.mscnn_kernel_launch_count()
        fn()
        return int(L.mscnn_kernel_launch_count() - n0)

    arms = {"single_class_x%d" % C: singles, "classes": classes}
    lc = {name: launches(fn) for name, fn in arms.items()}
    for _ in range(3):
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.reps)
    res = {}
    for name, t in times.items():
        a = np.array(t)
        res[name] = {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)),
                     "p90_ms": float(np.percentile(a, 90)), "launches_per_call": lc[name]}
    single = res["single_class_x%d" % C]["median_ms"]
    out = {"workload": f"final detections of kitti_ped_cyc/mscnn-8s-768-trainval, cls_ids {ids}, "
                       f"{B}x3x{H}x{W} synthetic, {net.num_proposals()} proposals",
           "card": card(), "rounds": args.rounds, "reps_per_round": args.reps, "arms": res,
           "detections_per_image_per_class": float(both[1].float().mean().item()),
           "speedup_median": single / res["classes"]["median_ms"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
