"""CPU side of the pedestrian-net checks (tests/test_pedestrian_layers_gpu.py, tests/test_pedestrian_nets_gpu.py):

* oracle.port's ROIPooling with 8x4 bins and BoxOutput with 1:2 anchors (field_w != field_h, with and without bbox
  normalisation) against the reference's own layers (test_oracle._ref_run: stored outputs of oracle/_ref, re-run
  live where it is built);
* port's BoxOutput on the fixtures' own LFCN maps reproduces the reference's proposals bit for bit;
* the fixtures of tests/golden/make_pedestrian_golden.py exist, stay under 1 MB and hold what the GPU tests read."""
from pathlib import Path

import numpy as np
import pytest

from oracle import port
from test_oracle import _ref_run

GOLD = Path(__file__).resolve().parent / "golden"
CALTECH = dict(field_w=[30, 42, 60, 84, 120, 168, 240], field_h=[60, 84, 120, 168, 240, 336, 480],
               downsample_rate=[8, 8, 16, 16, 32, 32, 64], fg_thr=-5.0, iou_thr=0.65, max_nms_num=2000)
CITYPERSONS = dict(field_w=[30, 42, 60, 84, 120, 168, 240, 336], field_h=[60, 84, 120, 168, 240, 336, 480, 672],
                   downsample_rate=[8, 8, 16, 16, 32, 32, 64, 64], fg_thr=-3.0, iou_thr=0.65, max_nms_num=2000,
                   bbox_mean=[0, 0, 0, 0], bbox_std=[0.1, 0.1, 0.2, 0.2])


def test_port_roi_pool_8x4_vs_reference_random():
    """pooled_h 8, pooled_w 4 at 1/8 and 1/4 with pad_ratio 0 and 0.25, on ROIs of the test_roi_pool_parity mix plus
    tall pedestrian boxes and boxes smaller than one bin."""
    rng = np.random.default_rng(84)
    n, c, h, w, r = 2, 16, 24, 40, 80
    x1, y1 = rng.uniform(-20, 300, r), rng.uniform(-20, 180, r)
    bw = rng.uniform(0.5, 120, r)
    bh = np.where(np.arange(r) % 2 == 0, 2.4 * bw, rng.uniform(0.5, 40, r))
    rois = np.stack([rng.integers(0, n, r), x1, y1, x1 + bw, y1 + bh], axis=1).astype(np.float32)
    rois[0] = [0, 1, 1, 10, 10]
    rois[1] = [1, 50, 40, 30, 20]
    rois[2] = [0, 500, 300, 600, 400]
    rois[3] = [1, 3.5, 4.5, 4.5, 5.5]
    variants = [(0.125, 0.0), (0.125, 0.25), (0.25, 0.0), (0.25, 0.25)]
    proto = f'input: "x" input_dim: {n} input_dim: {c} input_dim: {h} input_dim: {w}\n'
    proto += f'input: "r" input_dim: {r} input_dim: 5 input_dim: 1 input_dim: 1\n'
    for k, (s, pr) in enumerate(variants):
        proto += (f'layer {{ bottom: "x" bottom: "r" top: "o{k}" name: "o{k}" type: "ROIPooling" roi_pooling_param '
                  f'{{ pooled_w: 4 pooled_h: 8 spatial_scale: {s} pad_ratio: {pr} }} }}\n')
    x = rng.standard_normal((n, c, h, w)).astype(np.float32)
    out = _ref_run("roi_pool_8x4", proto, {"x": x, "r": rois.reshape(r, 5, 1, 1)}, [f"o{k}" for k in range(4)])
    for k, (s, pr) in enumerate(variants):
        got = port.roi_pool(x, rois, 8, 4, s, pr)
        assert got.shape == out[f"o{k}"].shape == (r, c, 8, 4)
        assert np.array_equal(got, out[f"o{k}"]), (s, pr)
        assert not np.array_equal(port.roi_pool(x, rois, 4, 8, s, pr).reshape(got.shape), got)


@pytest.mark.parametrize("net", ["caltech", "citypersons"])
def test_port_box_output_pedestrian_anchors_vs_reference_random(net):
    """The shipped box_output_param of each net (field_h = 2 field_w; CityPersons with bbox normalisation)."""
    p = CALTECH if net == "caltech" else CITYPERSONS
    rng = np.random.default_rng(len(net))
    j = len(p["field_w"])
    shapes = [(16, 24), (16, 24), (8, 12), (8, 12), (4, 6), (4, 6), (2, 3), (2, 3)][:j]
    proto = "".join(f'input: "m{k}" input_dim: 2 input_dim: 6 input_dim: {h} input_dim: {w}\n'
                    for k, (h, w) in enumerate(shapes))
    proto += "layer { " + " ".join(f'bottom: "m{k}"' for k in range(j)) + ' top: "r" top: "rs" name: "p" type: "BoxOutput" '
    proto += f'box_output_param {{ fg_thr: {p["fg_thr"]} iou_thr: 0.65 nms_type: "IOU" '
    proto += " ".join(f"field_w: {v}" for v in p["field_w"]) + " " + " ".join(f"field_h: {v}" for v in p["field_h"])
    proto += " " + " ".join(f"downsample_rate: {v}" for v in p["downsample_rate"]) + " field_whr: 2 field_xyr: 2 max_nms_num: 2000 }"
    if "bbox_std" in p:
        proto += " bbox_reg_param { " + " ".join(f"bbox_mean: {v}" for v in p["bbox_mean"]) + " "
        proto += " ".join(f"bbox_std: {v}" for v in p["bbox_std"]) + " }"
    proto += " }"
    maps = []
    for h, w in shapes:
        m = rng.standard_normal((2, 6, h, w)).astype(np.float32)
        m[:, :2] *= 3
        maps.append(m)
    out = _ref_run(f"box_output_{net}", proto, {f"m{k}": m for k, m in enumerate(maps)}, ["r", "rs"])
    rois, sc, _, count = port.box_output(maps, **p)
    assert count > 20
    assert np.array_equal(rois, out["r"].reshape(-1, 5))
    assert np.array_equal(sc, out["rs"].reshape(-1, 6))
    swapped, _, _, _ = port.box_output(maps, **dict(p, field_w=p["field_h"], field_h=p["field_w"]))
    assert swapped.shape != rois.shape or not np.array_equal(swapped, rois)


FIXTURES = {
    "e2e_caltech_7s_240x320.npz": (CALTECH, 7, (30, 40), ["conv4_3", "conv5_3", "conv6_1", "roi_pool", "roi_c1", "fc6"],
                                   ["cls_pred", "bbox_pred"]),
    "e2e_citypersons_cascade_192x384.npz": (
        CITYPERSONS, 8, (24, 48), ["conv4_3", "conv4_3_2x", "conv5_3", "conv6_1", "roi_pool", "roi_pool_2nd",
                                   "roi_pool_3rd", "fc6", "fc6_2nd", "fc6_3rd"],
        ["cls_pred", "bbox_pred", "proposals_2nd", "proposals_3rd", "output_bbox_1st", "output_bbox_2nd",
         "output_bbox_3rd", "cls_prob_1st", "cls_prob_2nd", "cls_prob_3rd", "cls_pred_2nd", "cls_pred_3rd",
         "bbox_pred_2nd", "bbox_pred_3rd", "cls_prob_1st_3rd", "cls_prob_2nd_3rd", "cls_prob_3rd_avg"]),
    "e2e_citypersons_8s_192x384.npz": (CITYPERSONS, 8, (24, 48), ["conv4_3", "conv4_3_2x", "conv5_3", "conv6_1",
                                                                   "roi_pool", "fc6"],
                                       ["cls_pred", "bbox_pred", "output_bbox_1st", "cls_prob_1st"]),
}


@pytest.mark.parametrize("name", list(FIXTURES))
def test_pedestrian_fixture_contents(name):
    p, nheads, first_map, subs, rows = FIXTURES[name]
    path = GOLD / name
    assert path.exists() and path.stat().st_size < 1_000_000, (name, path.stat().st_size if path.exists() else None)
    g = np.load(path)
    heads = sorted(k for k in g.files if k.startswith("LFCN_"))
    assert len(heads) == nheads
    for k, b in enumerate(heads):
        assert g[b].dtype == np.float32 and g[b].shape[:2] == (2, 6), b
        rate = p["downsample_rate"][k] // 8
        assert g[b].shape[2:] == (-(-first_map[0] // rate), -(-first_map[1] // rate)), (b, g[b].shape)
    r = g["proposals"].shape[0]
    assert r > 100 and g["proposals"].shape == (r, 5, 1, 1) and g["proposals_score"].shape == (r, 6, 1, 1)
    assert set(np.unique(g["proposals"][:, 0])) == {0.0, 1.0}
    for b in rows:
        assert g[b].shape[0] == r, b
    for b in subs:
        shape = tuple(g[b + "__shape"])
        assert g[b + "__sub"].shape == ((int(np.prod(shape)) + 7918) // 7919,) and g[b + "__m2"].shape == (1,), b
        if b.startswith("roi_pool"):
            assert shape == (r, 1024, 8, 4), (b, shape)
        if b.startswith("fc6"):
            assert shape == (r, 2048), (b, shape)


@pytest.mark.parametrize("name", ["e2e_caltech_7s_240x320.npz", "e2e_citypersons_8s_192x384.npz"])
def test_port_box_output_on_fixture_maps(name):
    """The reference's proposals of the fixture, from its own LFCN maps, are port.box_output's bit for bit: the
    oracle the GPU tests use agrees with the reference on real net outputs of 1:2 anchors."""
    p = FIXTURES[name][0]
    g = np.load(GOLD / name)
    maps = [g[b] for b in sorted(k for k in g.files if k.startswith("LFCN_"))]
    rois, sc, per, count = port.box_output(maps, **p)
    assert count == len(g["proposals"]) and per.sum() == count
    assert np.array_equal(rois, g["proposals"].reshape(-1, 5))
    assert np.array_equal(sc, g["proposals_score"].reshape(-1, 6))
