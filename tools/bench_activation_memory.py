"""Device memory and speed of a net with and without activation reuse (Net.set_activation_reuse).

For each configuration: the planned arena and the bytes without reuse (host plan), the device memory a net takes over
its first forward with reuse on and off (torch.cuda.mem_get_info around it; the weights belong to an owner net both
share, so only activations and per-net buffers count), and images/s with reuse on and off, alternated in one process
with the spread over rounds.  A configuration that does not fit the card is reported as such.  Prints one JSON line per
configuration and one with the card's name and power limit, read in the same process.

    python tools/bench_activation_memory.py [--rounds 3] [--steps 10] [--quick]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


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


def measure(name, proto, n, h, w, rounds, steps):
    import torch
    from mscnn_b200 import net as mnet, synth
    rec = {"config": name, "batch": n, "net_hw": [h, w]}
    if n * 64 * h * w >= 2 ** 31:        # conv1_1's top: a blob counts its values in an int, as Caffe's does
        rec["error"] = f"not measured: a blob of {n} x 64 x {h} x {w} values exceeds the blob's int count"
        return rec
    images = synth.make_images(n, h, w)
    owner = mnet.Net(proto)
    owner.set_params(synth.make_weights(owner.layers()))
    owner.set_activation_reuse(True)
    rec["planned_arena_bytes"], rec["planned_without_reuse_bytes"] = owner.activation_bytes()
    owner.set_input("data", images)
    owner.forward_only()             # uploads and packs the weights both measured nets share
    nets = {}
    try:
        for reuse in (True, False):
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            need = rec["planned_arena_bytes" if reuse else "planned_without_reuse_bytes"]
            if need + (2 << 30) > free0:     # a failed device allocation aborts the process: do not try
                rec[f"measured_bytes_{'on' if reuse else 'off'}"] = f"not measured: needs {need} B, {free0} B free"
                continue
            net = mnet.Net(proto)
            net.share_trained_layers_with(owner)
            if reuse:
                net.set_activation_reuse(True)
            net.set_input("data", images)
            net.forward_only()
            torch.cuda.synchronize()
            rec[f"measured_bytes_{'on' if reuse else 'off'}"] = free0 - torch.cuda.mem_get_info()[0]
            nets[reuse] = net
    except Exception as e:      # noqa: BLE001 -- reported, not measured
        rec["error"] = f"does not fit or failed: {e}"
        return rec
    del owner
    rates = {True: [], False: []}
    for _ in range(rounds):
        for reuse in nets:
            net = nets[reuse]
            net.forward_only()
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(steps):
                net.forward_only()
            torch.cuda.synchronize()
            rates[reuse].append(n * steps / (time.perf_counter() - t))
    for reuse in nets:
        r = rates[reuse]
        rec[f"images_per_s_{'on' if reuse else 'off'}"] = [round(float(np.median(r)), 2), round(min(r), 2),
                                                            round(max(r), 2)]
    if True in nets:
        rec["misses"] = nets[True].activation_misses()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--quick", action="store_true", help="small sizes only (a rehearsal)")
    a = ap.parse_args()
    import torch
    from mscnn_b200 import net as mnet, ops
    torch.cuda.init()
    print(json.dumps({"card": card()}), flush=True)
    mnet.set_precision("fp32")
    if a.quick:
        configs = [("kitti_8s", deploy("kitti_car/mscnn-8s-768-trainval", 2, 192, 640), 2, 192, 640)]
    else:
        configs = [("kitti_8s", deploy("kitti_car/mscnn-8s-768-trainval", 8, 768, 2560), 8, 768, 2560),
                   ("kitti_8s", deploy("kitti_car/mscnn-8s-768-trainval", 32, 768, 2560), 32, 768, 2560),
                   ("citypersons_cascade", deploy("citypersons/cascade-mscnn-8s-1344-2x", 8, 1344, 2688), 8, 1344,
                    2688)]
        # WIDER FACE at the net sizes tools/bench_widerface.py buckets its frames into (500 x 375 .. 1024 x 683)
        for oh, ow in ((375, 500), (683, 1024), (1024, 683)):
            h, w = ops.widerface_net_size(oh, ow, 0, 0, 3072)
            configs.append(("widerface", deploy("widerface/mscnn-12s-2x", 8, h, w), 8, h, w))
    for name, proto, n, h, w in configs:
        print(json.dumps(measure(name, proto, n, h, w, a.rounds, a.steps)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
