"""Timing of the convolution geometries beyond stride 1 / dilation 1 / group 1 and of global pooling (DESIGN.md 6), each
beside the plain layer of the same OUTPUT size, batch 8, in one process:

    stride 2, 3x3, 512 -> 512 at 96x320 (output 48x160)   vs  stride 1 at 48x160
    dilation 2, 3x3, 512 -> 512 at 48x160                 vs  dilation 1 at 48x160
    4 groups, 3x3, 512 -> 512 at 96x320                   vs  1 group at 96x320
    global AVE pooling of 512 x 24 x 80                   (GB/s of the planes read)

Rounds are interleaved: one round times every arm once (CUDA events around --iters launches), so drift of
the card's clocks hits all arms alike.  Prints one JSON object: per arm the median and the 10th / 90th percentile of the
per-launch time in ms, algorithmic TFLOP/s (2 N Ho Wo Cout Cin/g KH KW over the median; x3 MMAs are issued in
fp32-faithful mode, which this figure does not count) or GB/s, and the card's name, power limit and maximum SM clock read
in the same run.

    python tools/bench_conv_geometry.py [--rounds 9] [--iters 20] [--warmup 3]
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

N, C = 8, 512
# name: (H, W, pad, stride, dilation, group)
CONVS = {
    "stride2_96x320": (96, 320, 1, 2, 1, 1), "stride1_48x160": (48, 160, 1, 1, 1, 1),
    "dilation2_48x160": (48, 160, 2, 1, 2, 1),
    "group4_96x320": (96, 320, 1, 1, 1, 4), "group1_96x320": (96, 320, 1, 1, 1, 1),
}


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, plim, smax = [c.strip() for c in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax)}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None, "sm_max_mhz": None}


def percentile(xs: list[float], q: float) -> float:
    s = sorted(xs)
    return s[min(len(s) - 1, max(0, round(q * (len(s) - 1))))]


def measure(split: bool, rounds: int, iters: int, warmup: int) -> dict:
    import torch
    from mscnn_b200 import capi, ops
    g = torch.Generator(device="cpu").manual_seed(1706)
    arms = {}
    for name, (h, w, pad, stride, dil, group) in CONVS.items():
        x = ops.nchw_to_planes(torch.randn((N, C, h, w), generator=g).cuda(), split)
        wt = ops.pack_conv_weights((torch.randn((C, C // group, 3, 3), generator=g) * (2.0 * group / (C * 9)) ** 0.5).cuda(),
                                   torch.zeros(C).cuda(), split)
        y = ops.conv_forward(x, wt, pad, relu=True, stride=stride, dilation=dil, group=group)
        run = (lambda x=x, wt=wt, y=y, pad=pad, stride=stride, dil=dil, group=group:
               ops.conv_forward(x, wt, pad, relu=True, out=y, stride=stride, dilation=dil, group=group))
        flop = 2.0 * N * y.shape[1] * y.shape[2] * C * (C // group) * 9
        arms[name] = (run, {"flop": flop})
    xg = ops.nchw_to_planes(torch.randn((N, C, 24, 80), generator=g).cuda(), split)
    yg = ops.pool_forward(xg, None, 1, capi.POOL_AVE)
    arms["global_ave_24x80"] = (lambda: ops.pool_forward(xg, None, 1, capi.POOL_AVE, out=yg),
                                {"bytes": float(xg.hi.numel() * 2 * (2 if split else 1))})
    for run, _ in arms.values():
        for _ in range(warmup):
            run()
    torch.cuda.synchronize()
    samples = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (run, _) in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                run()
            b.record()
            b.synchronize()
            samples[name].append(a.elapsed_time(b) / iters)
    res = {}
    for name, xs in samples.items():
        med = statistics.median(xs)
        r = {"median_ms": round(med, 4), "p10_ms": round(percentile(xs, 0.1), 4), "p90_ms": round(percentile(xs, 0.9), 4)}
        work = arms[name][1]
        if "flop" in work:
            r["algorithmic_tflops"] = round(work["flop"] / (med * 1e-3) / 1e12, 1)
        else:
            r["gb_per_s"] = round(work["bytes"] / (med * 1e-3) / 1e9, 1)
        res[name] = r
    res["stride2_over_stride1"] = round(res["stride2_96x320"]["median_ms"] / res["stride1_48x160"]["median_ms"], 3)
    res["dilation2_over_dilation1"] = round(res["dilation2_48x160"]["median_ms"] / res["stride1_48x160"]["median_ms"], 3)
    res["group4_over_group1"] = round(res["group4_96x320"]["median_ms"] / res["group1_96x320"]["median_ms"], 3)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_conv_geometry.py needs a CUDA device"
    torch.cuda.set_device(0)
    out = {"workload": "3x3 512 -> 512 convolutions and global AVE pooling, batch 8, seeded", "rounds": args.rounds,
           "iters": args.iters, **card()}
    for precision, split in (("fp32", True), ("bf16", False)):
        out[precision] = measure(split, args.rounds, args.iters, args.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
