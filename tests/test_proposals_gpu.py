"""The drivers' proposal list on the device, and the CityPersons script's default net through the drivers.

(1) mscnn_proposals_postprocess / Net.proposals against tests/proposals_ref.py with exact float64 equality: hand-made
    rows (threshold ties, zero and -0.0 extents, NaN scores, quotients the fp32 ratio rounds differently, several
    compaction chunks), and the BoxOutput rows of the 8s net at 192x640, batch 8, mixed original KITTI sizes, read
    before the row count is resolved on the host, eager and as a CUDA graph, fp32-faithful and bf16.
(2) A batch of 8 equals eight batches of 1, bit for bit.
(3) A cap below what an image can carry is refused before any launch (no count written); the raw entry marks such an
    image with count -1.
(4) drivers.run(..., proposals=True) on one net and on two nets reusing activation memory: the same proposals, equal
    to the restatement of the one-image loop, and the same detections as proposals=False; widerface.run likewise at
    three net sizes.
(5) drivers.run with CITYPERSONS_BASELINE on citypersons/mscnn-8s-1344-2x at 192x384 against the one-image loop of
    Net.detect_cascade_classes(stage="1st"), its result file, and the device post-process of the golden first-stage
    blobs against the restated cascade post-process."""
import re
import tarfile
from pathlib import Path

import numpy as np
import pytest
import torch

import proposals_ref as R

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden"
NET_HW = (192, 640)
KITTI_ORG = [(375, 1242), (370, 1224), (374, 1238), (376, 1241), (375, 1242), (360, 1200), (370, 1224), (375, 1242)]


@pytest.fixture()
def side_stream(cuda):
    from mscnn_b200 import net as mnet
    s = torch.cuda.Stream()
    prev = torch.cuda.current_stream()
    torch.cuda.set_stream(s)
    mnet.set_stream(s.cuda_stream)
    yield s
    torch.cuda.synchronize()
    torch.cuda.set_stream(prev)
    mnet.set_stream(prev.cuda_stream)


def _frame(rng, h, w, gray=False):
    im = rng.integers(0, 256, size=(h, w) if gray else (h, w, 3), dtype=np.uint8)
    im[: h // 3, : w // 4] = 255
    return im


def _deploy(net, n, h, w):
    with tarfile.open(GOLD / "deploy.tar.xz") as t:
        text = t.extractfile(f"deploy/{net}/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: \d+\s+input_dim: \d+",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def _same(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _issue(net, cfg, n):
    """Net.proposals into fresh buffers (counts pre-set to -7); returns them, nothing synchronised."""
    props = torch.full((n, cfg.max_rois_per_image, 5), float("nan"), dtype=torch.float64, device="cuda")
    counts = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    net.proposals(cfg, props.data_ptr(), counts.data_ptr())
    return props, counts


def _read(props, counts):
    torch.cuda.synchronize()
    c, p = counts.cpu().numpy(), props.cpu().numpy()
    assert np.all(c >= 0), c
    return [p[i, :c[i]].copy() for i in range(len(c))]


def _expected(net, thr, net_hw, org):
    n = len(org)
    rows = R.split_rows(net.blob("proposals_score"), [net.num_proposals(i) for i in range(n)])
    return [R.proposals(rows[i], thr, net_hw, org[i]) for i in range(n)]


# -------------------------------------------------------------------------------------------- (1) hand-made rows
def test_kernel_on_hand_made_rows(cuda):
    from mscnn_b200 import net as mnet, ops
    rng = np.random.default_rng(7)
    z = np.float32(-0.0)
    x = np.float32(617.3)
    special = np.array([[0, 1, 2, 11, 22, -10.0], [0, 1, 2, 11, 22, np.nextafter(np.float32(-10), np.float32(-11))],
                        [0, 1, 2, 11, 22, np.nan], [0, 5, 5, 5, 9, 1], [0, 5, 5, 9, 5, 1], [0, 0, 5, z, 9, 1],
                        [0, 5, 0, 9, z, 1], [0, 5, 5, 4, 3, 1], [0, x, 0, x + 10, 10, 0]], dtype=np.float32)
    big = rng.uniform(0, 600, size=(700, 6)).astype(np.float32)          # three compaction chunks
    big[:, 3:5] = big[:, 1:3] + rng.choice([0.0, 3.5, -2.0, 40.0], size=(700, 2)).astype(np.float32)
    big[:, 5] = rng.normal(-9, 2, size=700).astype(np.float32)
    big[::37, 5] = np.nan
    big[:, 0] = 2
    per = [special, np.zeros((0, 6), np.float32), big, special[::-1]]
    rows = np.concatenate(per)
    org = np.array([[375, 1242], [100, 100], [384, 640], [370, 1224]], np.int32)
    num_out = torch.tensor([len(rows), len(rows)] + [len(p) for p in per], dtype=torch.int32, device=cuda)
    ps = torch.from_numpy(rows).to(cuda)
    for net_hw, thr in (((768, 2560), -10.0), ((192, 640), -9.0), ((768, 2560), float(np.float32(-8.765)))):
        cfg = mnet.kitti_detect_cfg(*net_hw)
        cfg.proposal_thr = thr
        props, counts = ops.proposals_postprocess(cfg, 4, ps, num_out, net_hw, org)
        got = _read(props, counts)
        for i in range(4):
            want = R.proposals(per[i], thr, net_hw, org[i])
            assert _same(got[i], want), (net_hw, thr, i)
        assert len(got[1]) == 0 and 0 < len(got[2]) < 700
    # the fp32-ratio quotient differs from the double one the kernel writes
    assert got[0][-1, 0] == float(x) / (2560 / 1242) != float(x) / float(np.float32(2560 / 1242))
    # org_hw NULL: the cfg's original size
    cfg = mnet.kitti_detect_cfg(768, 2560, org_hw=(375, 1242))
    props, counts = ops.proposals_postprocess(cfg, 4, ps, num_out, (768, 2560))
    got = _read(props, counts)
    for i in range(4):
        assert _same(got[i], R.proposals(per[i], -10.0, (768, 2560), (375, 1242))), i
    # more kept rows than cap: that image's count is -1, the others are untouched by it
    cfg = mnet.kitti_detect_cfg(192, 640)
    cfg.max_rois_per_image = 16
    props, counts = ops.proposals_postprocess(cfg, 4, ps, num_out, (192, 640), org)
    torch.cuda.synchronize()
    c = counts.cpu().numpy()
    assert c[2] == -1 and c[1] == 0 and c[0] == len(R.proposals(per[0], -10.0, (192, 640), org[0]))


# ------------------------------------------------------------------------------------------ (1) BoxOutput rows
@pytest.fixture(scope="module")
def kitti_weights(cuda):
    from mscnn_b200 import models, net as mnet, synth
    n = mnet.Net(models.kitti(*NET_HW, 8, False, batch=1))
    return synth.make_weights(n.layers())


def _kitti_frames(seed, k=8):
    rng = np.random.default_rng(seed)
    return [_frame(rng, *KITTI_ORG[i % len(KITTI_ORG)]) for i in range(k)]


@pytest.mark.parametrize("precision,graph", [("fp32", False), ("bf16", False), ("fp32", True), ("bf16", True)])
def test_net_proposals_equal_the_restatement(request, cuda, kitti_weights, precision, graph):
    from mscnn_b200 import models, net as mnet, ops
    if graph:
        request.getfixturevalue("side_stream")
    mnet.set_precision(precision)
    try:
        net = mnet.Net(models.kitti(*NET_HW, 8, False, batch=8))
        net.set_params(kitti_weights)
        net.set_graph(graph)
        pre = ops.Preprocess(KITTI_ORG[0], NET_HW)
        dropped = replays = 0
        for step, seed in enumerate((1, 2, 3)):
            frames = _kitti_frames(seed)
            org = [f.shape[:2] for f in frames]
            net.set_input_images("data", pre, frames)
            net.forward_only()
            replays += int(net.graph_replayed())
            cfg = mnet.kitti_detect_cfg(*NET_HW)
            issued = [(-10.0, _issue(net, cfg, 8))]                # before any host read: the row count is lazy
            cfg2 = mnet.kitti_detect_cfg(*NET_HW)                  # a threshold that drops about half the rows
            cfg2.proposal_thr = float(np.median(net.blob("proposals_score").reshape(-1, 6)[:, 5]))
            issued.append((cfg2.proposal_thr, _issue(net, cfg2, 8)))
            for thr, (props, counts) in issued:
                got = _read(props, counts)
                want = _expected(net, thr, NET_HW, org)
                for i in range(8):
                    assert _same(got[i], want[i]), (step, thr, i)
                total = sum(net.num_proposals(i) for i in range(8))
                dropped += total - sum(len(g) for g in got)
                assert sum(len(g) for g in got) > 0
        assert dropped > 0
        assert replays >= (1 if graph else 0)
    finally:
        mnet.set_precision("fp32")


def test_batch_of_8_equals_eight_batches_of_1(cuda, kitti_weights):
    from mscnn_b200 import models, net as mnet, ops
    mnet.set_precision("fp32")
    frames = _kitti_frames(4)
    net = mnet.Net(models.kitti(*NET_HW, 8, False, batch=8))
    net.set_params(kitti_weights)
    net.set_input_images("data", ops.Preprocess(KITTI_ORG[0], NET_HW), frames)
    net.forward_only()
    batch = _read(*_issue(net, mnet.kitti_detect_cfg(*NET_HW), 8))
    one = mnet.Net(models.kitti(*NET_HW, 8, False, batch=1))
    one.set_params(kitti_weights)
    for i, f in enumerate(frames):
        pre = ops.Preprocess(f.shape[:2], NET_HW)
        one.set_input_images("data", pre, f[None])         # an array batch records no sizes: the cfg's org_* apply
        one.forward_only()
        got, = _read(*_issue(one, mnet.kitti_detect_cfg(*NET_HW, org_hw=f.shape[:2]), 1))
        assert _same(got, batch[i]), i
    assert sum(len(b) for b in batch) > 0


# --------------------------------------------------------------------------------------------------- (3) the cap
def test_cap_below_box_output_rows_is_refused_before_any_launch(cuda, kitti_weights):
    from mscnn_b200 import capi, models, net as mnet, ops
    mnet.set_precision("fp32")
    net = mnet.Net(models.kitti(*NET_HW, 8, False, batch=2, max_nms_num=2000))
    net.set_params(kitti_weights)
    frames = _kitti_frames(5, 2)
    net.set_input_images("data", ops.Preprocess(KITTI_ORG[0], NET_HW), frames)
    net.forward_only()
    cfg = mnet.kitti_detect_cfg(*NET_HW, max_rois=1999)
    props = torch.zeros((2, 1999, 5), dtype=torch.float64, device=cuda)
    counts = torch.full((2,), -7, dtype=torch.int32, device=cuda)
    with pytest.raises(capi.MscnnError, match="max_rois_per_image"):
        net.proposals(cfg, props.data_ptr(), counts.data_ptr())
    torch.cuda.synchronize()
    assert counts.cpu().tolist() == [-7, -7] and not props.any()
    ok = _read(*_issue(net, mnet.kitti_detect_cfg(*NET_HW, max_rois=2000), 2))
    assert sum(len(p) for p in ok) > 0


# ------------------------------------------------------------------------------------------------ (4) the drivers
def _loop_proposals(net, frames, net_hw, thr, sized=None):
    """The drivers' loop: one frame per forward (at sized(h, w) when given), the proposal list restated from its
    proposals_score."""
    from mscnn_b200 import ops
    out = []
    for im in frames:
        im = np.repeat(im[:, :, None], 3, axis=2) if im.ndim == 2 else im
        oh, ow = im.shape[:2]
        hw = sized(oh, ow) if sized else net_hw
        if sized:
            net.reshape_input("data", 1, 3, *hw)
        pre = ops.Preprocess((oh, ow), hw)
        net.set_input_images("data", pre, im[None])
        net.forward_only()
        out.append(R.proposals(net.blob("proposals_score"), thr, hw, (oh, ow)))
    return out


def test_drivers_run_proposals_one_and_two_nets(cuda):
    from mscnn_b200 import drivers, net as mnet, synth
    mnet.set_precision("fp32")
    spec = drivers.KITTI_CAR
    proto = _deploy("kitti_car/mscnn-8s-768-trainval", 1, *NET_HW)
    rng = np.random.default_rng(9)
    sizes = [(120, 400), (110, 380), (125, 410), (100, 350)]
    frames = [_frame(rng, *sizes[k % 4], gray=(k % 5 == 3)) for k in range(12)]
    loop_net = mnet.Net(proto)
    weights = synth.make_weights(loop_net.layers())
    loop_net.set_params(weights)
    want = _loop_proposals(loop_net, frames, NET_HW, spec.proposal_thr)
    del loop_net
    net = mnet.Net(proto)
    net.set_params(weights)
    plain = drivers.run(net, frames, spec, batch=8, net_hw=NET_HW)
    dets, props = drivers.run(net, frames, spec, batch=8, net_hw=NET_HW, proposals=True)
    nets = drivers.make_nets(proto, weights, [0, 0], reuse_activations=True)
    dets2, props2 = drivers.run(nets, frames, spec, batch=4, net_hw=NET_HW, proposals=True)
    assert sum(len(p) for p in want) > 0
    for i in range(len(frames)):
        assert props[i].dtype == np.float64 and _same(props[i], want[i]), i
        assert _same(props2[i], want[i]), i
        for s in range(len(spec.cls_ids)):
            assert plain[i][s].tobytes() == dets[i][s].tobytes() == dets2[i][s].tobytes(), (i, s)


def test_widerface_run_proposals_at_three_net_sizes(cuda):
    from mscnn_b200 import models, net as mnet, ops, synth, widerface
    mnet.set_precision("fp32")
    org = [(120, 150), (100, 150), (130, 170), (150, 200), (90, 130)]
    rng = np.random.default_rng(2025)
    frames = [_frame(rng, *org[k % len(org)]) for k in range(8)]
    names = [f"img_{k}" for k in range(len(frames))]
    sized = lambda h, w: ops.widerface_net_size(h, w, 0, 0, widerface.MAX_SIZE)      # noqa: E731
    assert len({sized(*f.shape[:2]) for f in frames}) >= 3
    loop_net = mnet.Net(models.widerface(96, 128, batch=1))
    weights = synth.make_weights(loop_net.layers())
    loop_net.set_params(weights)
    want = _loop_proposals(loop_net, frames, None, -5.0, sized=sized)
    net = mnet.Net(models.widerface(96, 128, batch=1))
    net.set_params(weights)
    plain = widerface.run(net, frames, names)
    dets, props = widerface.run(net, frames, names, proposals=True)
    assert list(props) == names and sum(len(p) for p in want) > 0
    for k, name in enumerate(names):
        assert _same(props[name], want[k]), name
        assert dets[name].tobytes() == plain[name].tobytes(), name


# ------------------------------------------------------------------------------------------ (5) CityPersons 1st
def test_citypersons_baseline_driver(cuda, tmp_path):
    import detect_classes_ref as DR
    from mscnn_b200 import drivers, net as mnet, ops, synth
    mnet.set_precision("fp32")
    spec = drivers.CITYPERSONS_BASELINE
    net_hw = (192, 384)
    proto = _deploy("citypersons/mscnn-8s-1344-2x", 1, *net_hw)
    rng = np.random.default_rng(31)
    sizes = [(160, 320), (150, 300), (200, 400), (128, 256)]
    frames = [_frame(rng, *sizes[k % 4], gray=(k % 4 == 1)) for k in range(10)]
    loop_net = mnet.Net(proto)
    weights = synth.make_weights(loop_net.layers())
    loop_net.set_params(weights)
    want = []
    for im in frames:
        im3 = np.repeat(im[:, :, None], 3, axis=2) if im.ndim == 2 else im
        oh, ow = im3.shape[:2]
        loop_net.set_input_images("data", ops.Preprocess((oh, ow), net_hw), im3[None])
        loop_net.forward_only()
        cfg, classes = spec.detect_cfg(net_hw)
        geo = mnet.kitti_detect_cfg(*net_hw, org_hw=(oh, ow))
        cfg.ratio_h, cfg.ratio_w, cfg.org_h, cfg.org_w = geo.ratio_h, geo.ratio_w, geo.org_h, geo.org_w
        dets = torch.zeros((1, 1, cfg.max_rois_per_image, 5), device=cuda)
        cnt = torch.zeros((1, 1), dtype=torch.int32, device=cuda)
        loop_net.detect_cascade_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr(), stage="1st",
                                        cls_prob="cls_prob_1st")
        torch.cuda.synchronize()
        want.append([dets[0, 0, :int(cnt[0, 0])].cpu().numpy()])
    del loop_net
    net = mnet.Net(proto)
    net.set_params(weights)
    got = drivers.run(net, frames, spec, batch=4, net_hw=net_hw)
    assert sum(len(r[0]) for r in want) > 0
    for i in range(len(frames)):
        assert got[i][0].tobytes() == want[i][0].tobytes(), i
    a = drivers.write_results(tmp_path / "loop", spec, "mscnn_8s_1344_2x_pretrained", [want[:4], want[4:]], groups=True)
    b = drivers.write_results(tmp_path / "run", spec, "mscnn_8s_1344_2x_pretrained", [got[:4], got[4:]], groups=True)
    assert [p.name for p in b] == ["mscnn_8s_1344_2x_pretrained_1st_results.txt"]
    assert a[0].read_bytes() == b[0].read_bytes() and b[0].stat().st_size > 0

    # the device post-process of the golden first-stage blobs against the restated run_cascademscnn.m lines
    g = np.load(GOLD / "e2e_citypersons_8s_192x384.npz")
    props = g["proposals"].reshape(-1, 5)
    prob = g["cls_prob_1st"].reshape(len(props), -1)
    outb = g["output_bbox_1st"].reshape(-1, 5)
    n = int(props[:, 0].max()) + 1
    per = [int((props[:, 0] == i).sum()) for i in range(n)]
    assert sum(per) == len(props) and n == 2
    org = [(384, 768), (300, 500)]
    geom = mnet.image_geometry((192, 384), org)
    cfg, classes = spec.detect_cfg((192, 384))
    num_out = torch.tensor([len(props), len(props)] + per, dtype=torch.int32, device=cuda)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)          # noqa: E731
    dets, cnt = ops.cascade_detect_postprocess_classes(cfg, classes, n, t(props), t(prob), t(outb), num_out, geom)
    torch.cuda.synchronize()
    dets, cnt = dets.cpu().numpy(), cnt.cpu().numpy()
    start = 0
    for i in range(n):
        sl = slice(start, start + per[i])
        ref, = DR.cascade_detect_postprocess_classes(props[sl], prob[sl], outb[sl], [2], overlap=cfg.nms_overlap,
                                                     ratios=(geom[i, 0], geom[i, 1]), org_hw=(geom[i, 2], geom[i, 3]))
        assert cnt[i, 0] == len(ref), (i, cnt[i, 0], len(ref))
        np.testing.assert_allclose(dets[i, 0, :cnt[i, 0]], ref, rtol=1e-5, atol=1e-5)
        start = sl.stop
    assert cnt.sum() > 0
