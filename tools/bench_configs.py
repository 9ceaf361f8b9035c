"""The other single-GPU configurations BASELINE.json lists (bench.py measures configs[2]); same protocol as bench.py's
`value` (inputs resident in HBM, one step = forward of the batch + final-detection post-process, CUDA events):

    configs[1]  mscnn-7s-576-2x full detection forward (conv4_3_2x deconvolution, ROI scale 1/4), batch 1, 3x576x1920
    configs[4]  WIDER FACE mscnn-12s-2x, 3x768x1024, batch 8 (12 proposal heads, 3000-box NMS)

Prints one JSON object with both, fp32-faithful and plain bf16.  python tools/bench_configs.py [--steps 10] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def run(name, proto, H, W, B, cfg, steps, warmup):
    import torch
    from mscnn_b200 import capi, net as mnet, synth
    dev = torch.device("cuda", 0)
    out = {"workload": name, "batch": B}
    for mode in ("fp32", "bf16"):
        mnet.set_precision(mode)
        net = mnet.Net(proto)
        net.set_params(synth.make_weights(net.layers()))
        img = torch.from_numpy(synth.make_images(B, H, W)).to(dev)
        cap = cfg.max_rois_per_image
        dets = torch.zeros((B, cap, 5), device=dev)
        cnt = torch.zeros(B, dtype=torch.int32, device=dev)

        def step():
            net.set_input("data", img)
            net.forward_only()
            net.detect(cfg, dets.data_ptr(), cnt.data_ptr())

        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        n0 = capi.lib().mscnn_kernel_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        launches = (capi.lib().mscnn_kernel_launch_count() - n0) // steps
        # the same loop with whole forwards replayed as ONE CUDA graph launch (Net.set_graph; the first forward after
        # switching it on runs eagerly, the second is captured, later ones are replays)
        net.set_graph(True)
        for _ in range(max(warmup, 3)):
            step()
        torch.cuda.synchronize()
        replayed = net.graph_replayed()
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms_graph = e0.elapsed_time(e1) / steps
        net.set_graph(False)
        lt = net.time_layers()
        out["fp32_faithful" if mode == "fp32" else "bf16"] = {
            "ms_per_step": ms, "value": B / (ms / 1e3), "unit": "images/s",
            "graph": {"ms_per_step": ms_graph, "value": B / (ms_graph / 1e3), "replayed": bool(replayed)},
            "proposals_per_image": net.num_proposals() / B, "detections_per_image": float(cnt.float().mean().item()),
            "kernel_launches_per_step": launches,
            "layers_ms_sum": round(sum(lt.values()), 3),
            "top_layers_ms": sorted(((round(v, 3), k) for k, v in lt.items()), reverse=True)[:12]}
        del net
    mnet.set_precision("fp32")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from mscnn_b200 import models, net as mnet
    torch.cuda.set_device(0)
    mnet.set_device(0)
    side = torch.cuda.Stream()          # a CUDA graph cannot be captured on the legacy default stream
    torch.cuda.set_stream(side)
    mnet.set_stream(side.cuda_stream)
    res = {"n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic (mscnn_b200/synth.py, seed 1706)"}
    cfg = mnet.kitti_detect_cfg(576, 1920)
    res["config1"] = run("mscnn-7s-576-2x full detection forward, 1x3x576x1920 (BASELINE.json configs[1])",
                         models.kitti(576, 1920, 7, True, batch=1), 576, 1920, 1, cfg, args.steps, args.warmup)
    wcfg, _ = mnet.widerface_detect_cfg(768, 1024)         # net.detect: class 2 alone, without det_thr
    res["config4"] = run("WIDER FACE mscnn-12s-2x forward, 8x3x768x1024 (BASELINE.json configs[4])",
                         models.widerface(768, 1024, batch=8), 768, 1024, 8, wcfg, args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
