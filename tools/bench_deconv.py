"""Timing of Deconvolution (DESIGN.md 6), batch 8, in one process, each dense arm beside the convolution with the same
MMA count:

    dense 512 -> 512, k4 / s2 / p1, input 48x160 (output 96x320)   vs  2x2 convolution, stride 1, output 96x320
    dense 256 -> 256, k2 / s2 / p0, input 96x320 (output 192x640)  vs  1x1 convolution at 192x640
    depthwise 512, the shipped k4 / s2 / p1 layer (mscnn_deconv2x_forward) and k8 / s4 / p2, input 48x160

Rounds are interleaved: one round times every arm once (CUDA events around --iters launches), so drift of the card's
clocks hits all arms alike.  Prints one JSON object: per arm the median and the 10th / 90th percentile of the
per-launch time in ms (a deconvolution launch = all of its phases), algorithmic TFLOP/s (2 N H W Cin Cout/g KH KW over
the median; fp32-faithful mode issues 3x the MMAs, which this figure does not count) or GB/s of planes read and written,
the deconvolution / convolution time ratios, and the card's name, power limit and maximum SM clock read in the same
run.  --profile adds, per precision, the CUDA kernel times of the dense arms from torch.profiler (a separate pass).

    python tools/bench_deconv.py [--rounds 9] [--iters 20] [--warmup 3] [--profile]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tools")]

from bench_conv_geometry import card, percentile  # noqa: E402

N = 8


def arms(split: bool) -> dict:
    import torch
    from mscnn_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(1706)
    out = {}

    def deconv(name, c, h, w, k, s, p):
        x = ops.nchw_to_planes(torch.randn((N, c, h, w), generator=g).cuda(), split)
        wt = (torch.randn((c, c, k, k), generator=g) * (2.0 / (c * k * k)) ** 0.5).cuda()
        wp = ops.pack_deconv_weights(wt, torch.zeros(c).cuda(), split, s, p)
        y = ops.deconv_forward(x, wp)
        out[name] = (lambda: ops.deconv_forward(x, wp, out=y), {"flop": 2.0 * N * h * w * c * c * k * k})

    def conv(name, c, h, w, k):
        x = ops.nchw_to_planes(torch.randn((N, c, h, w), generator=g).cuda(), split)
        wp = ops.pack_conv_weights((torch.randn((c, c, k, k), generator=g) * (2.0 / (c * k * k)) ** 0.5).cuda(),
                                   torch.zeros(c).cuda(), split)
        y = ops.conv_forward(x, wp, 0, relu=False)
        out[name] = (lambda: ops.conv_forward(x, wp, 0, relu=False, out=y),
                     {"flop": 2.0 * N * y.shape[1] * y.shape[2] * c * c * k * k})

    deconv("deconv512_k4s2p1_48x160", 512, 48, 160, 4, 2, 1)
    conv("conv512_k2_96x320", 512, 97, 321, 2)
    deconv("deconv256_k2s2_96x320", 256, 96, 320, 2, 2, 0)
    conv("conv256_k1_192x640", 256, 192, 640, 1)
    planes = 2 if split else 1
    x = ops.nchw_to_planes(torch.randn((N, 512, 48, 160), generator=g).cuda(), split)
    w4 = torch.randn((512, 1, 4, 4), generator=g).cuda()
    w8 = torch.randn((512, 1, 8, 8), generator=g).cuda()
    ops.deconv2x_forward(x, w4)
    ops.deconv_depthwise_forward(x, w8, None, 4, 2)
    moved = lambda up: float(x.hi.numel() * 2 * planes * (1 + up * up))   # noqa: E731
    out["depthwise512_k4s2p1_48x160"] = (lambda: ops.deconv2x_forward(x, w4), {"bytes": moved(2)})
    out["depthwise512_k8s4p2_48x160"] = (lambda: ops.deconv_depthwise_forward(x, w8, None, 4, 2), {"bytes": moved(4)})
    return out


def measure(split: bool, rounds: int, iters: int, warmup: int) -> dict:
    import torch
    runs = arms(split)
    for run, _ in runs.values():
        for _ in range(warmup):
            run()
    torch.cuda.synchronize()
    samples = {k: [] for k in runs}
    for _ in range(rounds):
        for name, (run, _) in runs.items():
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
        work = runs[name][1]
        if "flop" in work:
            r["algorithmic_tflops"] = round(work["flop"] / (med * 1e-3) / 1e12, 1)
        else:
            r["gb_per_s"] = round(work["bytes"] / (med * 1e-3) / 1e9, 1)
        res[name] = r
    res["conv_over_deconv_512_k4s2"] = round(res["conv512_k2_96x320"]["median_ms"] /
                                             res["deconv512_k4s2p1_48x160"]["median_ms"], 3)
    res["conv_over_deconv_256_k2s2"] = round(res["conv256_k1_192x640"]["median_ms"] /
                                             res["deconv256_k2s2_96x320"]["median_ms"], 3)
    return res


def profile(split: bool, iters: int) -> dict:
    """CUDA time per kernel name over `iters` launches of each dense arm (torch.profiler, its own pass)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    runs = arms(split)
    out = {}
    for name in ("deconv512_k4s2p1_48x160", "conv512_k2_96x320", "deconv256_k2s2_96x320", "conv256_k1_192x640"):
        run = runs[name][0]
        run()
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                run()
            torch.cuda.synchronize()
        kernels = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                k = kernels.setdefault(ev.name[:60], [0, 0.0])
                k[0] += 1
                k[1] += ev.device_time / 1e3
        out[name] = {k: {"launches_per_call": c / iters, "ms_per_call": round(t / iters, 4)} for k, (c, t) in kernels.items()}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_deconv.py needs a CUDA device"
    torch.cuda.set_device(0)
    out = {"workload": "deconvolutions beside convolutions of the same MMA count, batch 8, seeded", "rounds": args.rounds,
           "iters": args.iters, **card()}
    for precision, split in (("fp32", True), ("bf16", False)):
        out[precision] = measure(split, args.rounds, args.iters, args.warmup)
    if args.profile:
        for precision, split in (("fp32", True), ("bf16", False)):
            out[f"{precision}_kernels"] = profile(split, 5)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
