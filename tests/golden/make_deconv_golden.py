"""Writes tests/golden/deconv_net.npz: every blob of tests/deconv_ref.deconv_net computed by the reference's
own CPU layers (oracle/_ref, built where the reference sources are mounted) at the two input sizes of DECONV_SIZES,
on mscnn_b200.synth's seeded weights and images.  tests/test_deconv_gpu.py reads only the fixture.

    python tests/golden/make_deconv_golden.py
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

from deconv_ref import DECONV_BLOBS, DECONV_SIZES, deconv_net  # noqa: E402
from mscnn_b200 import synth  # noqa: E402
from mscnn_b200.net import Net  # noqa: E402
from oracle import ref  # noqa: E402


def main():
    out = {}
    h0, w0 = DECONV_SIZES[0]
    weights = synth.make_weights(Net(deconv_net(h0, w0)).layers())
    for h, w in DECONV_SIZES:
        net = ref.RefNet(deconv_net(h, w))
        net.set_params(weights)
        net.set_blob("data", synth.make_images(2, h, w))
        net.forward()
        for b in DECONV_BLOBS:
            out[f"{h}x{w}/{b}"] = net.blob(b)
    np.savez_compressed(Path(__file__).with_name("deconv_net.npz"), **out)


if __name__ == "__main__":
    main()
