"""Generate tests/golden/e2e_pedcyc_8s_192x640.npz from oracle/_ref -- the reference's own CPU layer code compiled
verbatim (oracle/build_ref.py).  Run where /root/reference is mounted:

    python tests/golden/make_pedcyc_golden.py

The net is the shipped KITTI pedestrian / cyclist deploy file kitti_ped_cyc/mscnn-8s-768-trainval (from
tests/golden/deploy.tar.xz: eight 7-channel heads, cls_pred 3, bbox_pred 12) with its input set to 2x3x192x640,
synthetic seeded weights and images (mscnn_b200/synth.py).  Kept, as in the car twin e2e_8s_192x640.npz written by
make_golden.py: the eight LFCN maps, proposals, proposals_score, cls_pred, bbox_pred and a fixed sub-sample (stride
7919) with the second moment of the trunk, ROI-pooling and fc6 blobs.
"""
import re
import sys
import tarfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np  # noqa: E402

from make_golden import OUT, run_net  # noqa: E402


def pedcyc_deploy(n: int, h: int, w: int) -> str:
    """The shipped kitti_ped_cyc/mscnn-8s-768-trainval deploy file with its input set to n x 3 x h x w."""
    with tarfile.open(OUT / "deploy.tar.xz") as t:
        text = t.extractfile("deploy/kitti_ped_cyc/mscnn-8s-768-trainval/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: 768\s+input_dim: 2560",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def main():
    heads8 = [f"LFCN_{i}_{k}" for i in (1, 2, 3, 4) for k in ("3x5", "5x7")]
    g = run_net(pedcyc_deploy(2, 192, 640), 2, 192, 640,
                keep=heads8 + ["proposals", "proposals_score", "cls_pred", "bbox_pred"],
                sub=["conv1_2", "conv2_2", "conv3_3", "conv4_3", "conv5_3", "conv6_1", "roi_pool", "fc6"])
    np.savez_compressed(OUT / "e2e_pedcyc_8s_192x640.npz", **g)
    print("e2e_pedcyc_8s_192x640: proposals", g["proposals"].shape)


if __name__ == "__main__":
    main()
