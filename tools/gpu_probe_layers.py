"""Micro-timings of individual layers at the bench shapes (batch 8, mscnn-8s-768) with CUDA events.
Variants are toggled through the environment (read per call by the native code)."""
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch

from mscnn_b200 import ops


def timeit(fn, iters=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    dev = torch.device("cuda:0")
    B = 8
    for name, cin, h, w, cout in [("conv1_2", 64, 768, 2560, 64), ("conv2_1", 64, 384, 1280, 128), ("conv2_2", 128, 384, 1280, 128)]:
        xin = torch.randn((B, cin, h, w), device=dev)
        wt = torch.randn((cout, cin, 3, 3), device=dev) * (2.0 / (cin * 9)) ** 0.5
        for split in (True, False):
            xp = ops.nchw_to_planes(xin, split)
            wp = ops.pack_conv_weights(wt, None, split)
            msg = f"{name} split={split}:"
            for fat in ((False, True) if split else (False,)):
                if fat:
                    os.environ.pop("MSCNN_NO_FAT", None)
                else:
                    os.environ["MSCNN_NO_FAT"] = "1"
                ops.reload_config()
                t = timeit(lambda: ops.conv_forward(xp, wp, 1, relu=True))
                msg += f"  {'fat' if fat else 'term-major'} {t:.3f}"
            os.environ.pop("MSCNN_NO_FAT", None)
            ops.reload_config()
            t = timeit(lambda: ops.conv_forward(xp, wp, 1, relu=True))
            msg += f"  default {t:.3f} ms"
            flops = 2.0 * B * cin * cout * 9 * h * w
            print(msg + f"  ({flops / t / 1e9:.0f} TFLOP/s algorithmic)", flush=True)
            del xp, wp
        del xin


if __name__ == "__main__":
    main()
