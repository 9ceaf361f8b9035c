"""A/B timing of the row-share delivery of the narrow trunk convolutions (conv1_2, conv2_1, conv2_2; DESIGN.md 4.1c)
in ONE process: the bench net (mscnn-8s, batch 8, 3x768x2560, seeded weights and images) with MSCNN_NO_ROWSHARE=1
(one activation tile per tap) and unset (one haloed tile per three taps), alternated for --rounds rounds of
Net.time_layers() (per-layer CUDA events), in fp32-faithful and in plain bf16.

Prints one JSON object: per layer and arm the median and max-min spread in ms, the same for the three layers' sum and
for the whole step (sum of all layers), plus the card's name, power limit and maximum SM clock read in the same run.

    python tools/bench_rowshare.py [--rounds 5] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

NARROW = ("conv1_2", "conv2_1", "conv2_2")
ARMS = {"per_tap": {"MSCNN_NO_ROWSHARE": "1"}, "rowshare": {}}


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, plim, smax = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax)}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None, "sm_max_mhz": None}


def set_arm(env: dict) -> None:
    from mscnn_b200 import ops
    os.environ.pop("MSCNN_NO_ROWSHARE", None)
    os.environ.update(env)
    ops.reload_config()


def stats(xs: list[float]) -> dict:
    return {"median": round(statistics.median(xs), 3), "spread": round(max(xs) - min(xs), 3),
            "runs": [round(x, 3) for x in xs]}


def measure(precision: str, rounds: int, warmup: int) -> dict:
    import torch
    from mscnn_b200 import models, net as mnet, synth
    mnet.set_precision(precision)
    net = mnet.Net(models.kitti(768, 2560, 8, False, batch=8))
    net.set_params(synth.make_weights(net.layers()))
    net.set_input("data", torch.from_numpy(synth.make_images(8, 768, 2560)).cuda())
    for env in ARMS.values():               # warm every plan and module of both arms
        set_arm(env)
        for _ in range(warmup):
            net.forward_only()
    torch.cuda.synchronize()
    samples = {arm: [] for arm in ARMS}
    for _ in range(rounds):
        for arm, env in ARMS.items():
            set_arm(env)
            net.forward_only()
            samples[arm].append(net.time_layers())
    set_arm({})
    del net
    mnet.set_precision("fp32")
    res = {}
    for arm, runs in samples.items():
        r = {k: stats([t[k] for t in runs]) for k in NARROW}
        r["narrow_sum"] = stats([sum(t[k] for k in NARROW) for t in runs])
        r["step_sum"] = stats([sum(t.values()) for t in runs])
        res[arm] = r
    a, b = res["per_tap"]["narrow_sum"]["median"], res["rowshare"]["narrow_sum"]["median"]
    res["narrow_sum_change"] = round(b / a - 1.0, 4)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from mscnn_b200 import net as mnet
    assert torch.cuda.is_available(), "bench_rowshare.py needs a CUDA device"
    torch.cuda.set_device(0)
    mnet.set_device(0)
    mnet.set_stream(torch.cuda.current_stream().cuda_stream)
    out = {"workload": "mscnn-8s-768, batch 8, 3x768x2560 synthetic", "rounds": args.rounds, **card()}
    for precision in ("fp32", "bf16"):
        out[precision] = measure(precision, args.rounds, args.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
