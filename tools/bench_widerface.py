"""The WIDER FACE drivers' workload: every image at its own net size (examples/widerface/run_mscnn_detection.m:70-81).
Two arms over the same frames on one mscnn-12s-2x net (synthetic weights, mscnn_b200/synth.py):

    bucketed  widerface.run: images grouped by net size, batches of up to 8 (pixel budget 8 x 768 x 2560)
    loop      the drivers' loop: one frame per forward, in input order, the net reshaped to each frame's size

Both arms pre-process on the device (ops.Preprocess plans cached per net size) and end with the kept detections on the
host.  The frames are a seeded synthetic set of WIDER-like sizes: widths 1024, heights spread so that there are several
net sizes, some above 2048.  The two arms' result lists must be identical (checked before any time is reported); the
arms alternate within one process, and the median and spread over the rounds are reported as images/s, with the card's
name and power limit.

    python tools/bench_widerface.py [--images 32] [--rounds 3] [--precision fp32|bf16]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

HEIGHTS = [576, 683, 768, 1024, 1366]      # landscape and portrait frames 1024 wide
TALL = [2200, 2600]                        # net heights above 2048 (2208, 2592)


def wider_sizes(n: int, seed: int = 1706) -> list[tuple[int, int]]:
    rng = np.random.default_rng(seed)
    return [(int(rng.choice(TALL)) if i % 8 == 7 else int(rng.choice(HEIGHTS)), 1024) for i in range(n)]


def card() -> dict:
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit": "unknown"}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        if r.returncode == 0 and r.stdout.strip():
            out["power_limit"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pass
    return out


def driver_loop(net, frames, names, plans):
    """One frame per forward, each at its own net size (run_mscnn_detection.m:68-146)."""
    import torch
    from mscnn_b200 import net as mnet, ops
    out = {}
    for name, im in zip(names, frames):
        rz = ops.widerface_net_size(im.shape[0], im.shape[1], 0, 0, 3072)
        net.reshape_input("data", 1, 3, *rz)
        pre = plans.get(rz)
        if pre is None:
            pre = plans[rz] = ops.Preprocess(im.shape[:2], rz)
        net.set_input_images("data", pre, [im])
        net.forward_only()
        cfg, classes = mnet.widerface_detect_cfg(*rz)
        dets = torch.empty((1, 1, cfg.max_rois_per_image, 5), dtype=torch.float32, device="cuda")
        cnt = torch.empty((1, 1), dtype=torch.int32, device="cuda")
        net.detect_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr())
        out[name] = dets[0, 0, :int(cnt[0, 0])].cpu().numpy()
    return out


def same(a: dict, b: dict) -> bool:
    return list(a) == list(b) and all(a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes() for k in a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", choices=("fp32", "bf16"), default="fp32")
    args = ap.parse_args()
    import torch
    from mscnn_b200 import models, net as mnet, synth, widerface
    if not torch.cuda.is_available():
        sys.exit("bench_widerface.py needs a CUDA device")
    torch.cuda.set_device(0)
    mnet.set_device(0)
    mnet.set_precision(args.precision)
    sizes = wider_sizes(args.images)
    rng = np.random.default_rng(1706)
    frames = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
    names = [f"0_Parade_marchingband_1_{i}" for i in range(len(frames))]
    net = mnet.Net(models.widerface(768, 1024, batch=1))
    net.set_params(synth.make_weights(net.layers()))
    plans_b, plans_l = {}, {}
    arms = {"bucketed": lambda: widerface.run(net, frames, names, plans=plans_b),
            "loop": lambda: driver_loop(net, frames, names, plans_l)}
    ref = arms["bucketed"]()                   # warm-up of every shape, and the results both arms must give
    if not same(arms["loop"](), ref):
        sys.exit("bench_widerface.py: the bucketed run and the driver loop disagree")
    times = {k: [] for k in arms}
    for r in range(args.rounds):
        for k in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = arms[k]()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
            if not same(res, ref):
                sys.exit(f"bench_widerface.py: arm {k} changed its results in round {r}")
    n = len(frames)
    out = {"card": card(), "precision": args.precision, "images": n, "rounds": args.rounds,
           "net_sizes": sorted({hw for hw, _ in widerface.plan_batches(sizes)}, reverse=True),
           "batches": len(widerface.plan_batches(sizes)),
           "detections": int(sum(len(v) for v in ref.values()))}
    for k, t in times.items():
        med = float(np.median(t))
        out[k] = {"images_per_s": n / med, "median_s": med, "min_s": float(min(t)), "max_s": float(max(t))}
    out["speedup"] = out["bucketed"]["images_per_s"] / out["loop"]["images_per_s"]
    print(f"{out['card']['name']}, power limit {out['card']['power_limit']}, {args.precision}, {n} images, "
          f"{len(out['net_sizes'])} net sizes in {out['batches']} batches")
    for k in times:
        print(f"  {k:9s} {out[k]['images_per_s']:8.2f} images/s  (median {out[k]['median_s']:.3f} s, "
              f"min {out[k]['min_s']:.3f}, max {out[k]['max_s']:.3f})")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
