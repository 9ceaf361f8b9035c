"""Generate the pedestrian-net golden vectors from oracle/_ref -- the reference's own CPU layer code compiled verbatim
(oracle/build_ref.py).  Run where /root/reference is mounted:

    python tests/golden/make_pedestrian_golden.py

The nets are the shipped deploy files the Caltech and CityPersons drivers run (from tests/golden/deploy.tar.xz), with
only their input reshaped, synthetic seeded weights and images (mscnn_b200/synth.py).  Their geometry is the one no
other fixture has: 1:2 anchors (field_h = 2 field_w), heads of 5x3 and 7x5 kernels with 6 outputs, and 8x4 ROI bins.

  e2e_caltech_7s_240x320.npz   caltech/mscnn-7s-720 at 2x3x240x320 (the driver's 720x960 is 3:4 too): seven LFCN maps,
                               BoxOutput without bbox normalisation, ROIPooling at 1/8 on conv4_3.
  e2e_citypersons_cascade_192x384.npz  citypersons/cascade-mscnn-8s-1344-2x at 2x3x192x384: eight LFCN maps, three
                               ROIPooling stages at 1/4 on conv4_3_2x, every stage's boxes and probabilities and the
                               Eltwise average cls_prob_3rd_avg.
  e2e_citypersons_8s_192x384.npz  citypersons/mscnn-8s-1344-2x at 2x3x192x384: the single-stage net (DecodeBBox, Softmax).

Kept as in the other e2e fixtures (make_golden.py): the LFCN maps and the head outputs in full, and a fixed sub-sample
(stride 7919) with the second moment and the shape of the trunk, ROI-pooling and fc6 blobs.  The reference forward is
deterministic, so a second run rewrites the same arrays.
"""
import re
import sys
import tarfile
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent))
import numpy as np  # noqa: E402

from make_golden import OUT, run_net  # noqa: E402

TRUNK = ["conv1_2", "conv2_2", "conv3_3", "conv4_3", "conv5_3", "conv6_1"]
HEADS_7 = [f"LFCN_{i}_{k}" for i in (1, 2, 3) for k in ("3x5", "5x7")] + ["LFCN_4_3x5"]
HEADS_8 = [f"LFCN_{i}_{k}" for i in (1, 2, 3, 4) for k in ("3x5", "5x7")]
STAGES = ["proposals", "proposals_score", "proposals_2nd", "proposals_3rd", "output_bbox_1st", "output_bbox_2nd",
          "output_bbox_3rd", "cls_prob_1st", "cls_prob_2nd", "cls_prob_3rd", "cls_pred", "cls_pred_2nd", "cls_pred_3rd",
          "bbox_pred", "bbox_pred_2nd", "bbox_pred_3rd", "cls_prob_1st_3rd", "cls_prob_2nd_3rd", "cls_prob_3rd_avg"]


def shipped_deploy(net: str, n: int, h: int, w: int) -> str:
    """deploy/<net>/mscnn_deploy.prototxt from tests/golden/deploy.tar.xz with its input set to n x 3 x h x w."""
    with tarfile.open(OUT / "deploy.tar.xz") as t:
        text = t.extractfile(f"deploy/{net}/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: \d+\s+input_dim: \d+",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def main():
    g = run_net(shipped_deploy("caltech/mscnn-7s-720", 2, 240, 320), 2, 240, 320,
                keep=HEADS_7 + ["proposals", "proposals_score", "cls_pred", "bbox_pred"],
                sub=TRUNK + ["roi_pool", "roi_c1", "fc6"])
    np.savez_compressed(OUT / "e2e_caltech_7s_240x320.npz", **g)
    print("e2e_caltech_7s_240x320: proposals", g["proposals"].shape)
    g = run_net(shipped_deploy("citypersons/cascade-mscnn-8s-1344-2x", 2, 192, 384), 2, 192, 384,
                keep=HEADS_8 + STAGES,
                sub=TRUNK + ["conv4_3_2x", "roi_pool", "roi_pool_2nd", "roi_pool_3rd", "fc6", "fc6_2nd", "fc6_3rd"])
    np.savez_compressed(OUT / "e2e_citypersons_cascade_192x384.npz", **g)
    print("e2e_citypersons_cascade_192x384: proposals", g["proposals"].shape)
    g = run_net(shipped_deploy("citypersons/mscnn-8s-1344-2x", 2, 192, 384), 2, 192, 384,
                keep=HEADS_8 + ["proposals", "proposals_score", "cls_pred", "bbox_pred", "output_bbox_1st",
                                "cls_prob_1st"],
                sub=TRUNK + ["conv4_3_2x", "roi_pool", "fc6"])
    np.savez_compressed(OUT / "e2e_citypersons_8s_192x384.npz", **g)
    print("e2e_citypersons_8s_192x384: proposals", g["proposals"].shape)


if __name__ == "__main__":
    main()
