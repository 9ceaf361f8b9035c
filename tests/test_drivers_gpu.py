"""Gray frames, pre-processing of the next batch during a forward, and the fixed-size driver runners, on the GPU.

(a) Gray frames ([h][w] / [h][w][1]) through the device pre-processing give bit for bit what their repmat to three
    channels gives: arrays, lists, device lists, a batch mixing gray and colour frames of several sizes, and the full
    375x1242 -> 768x2560 size.
(b) Net.set_input_images_async, issued while the previous forward is in flight, over batches of changing original
    sizes: every batch's input blob and final detections equal those of the synchronous sequence, eager and graph.
(c) drivers.run for the five specs against the drivers' one-image loop built from the existing calls
    (set_input_images of one frame, forward_only, detect_classes / detect_cascade_classes): every image's detections
    and the written files are bit-identical."""
import re
import tarfile
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden"


def _repmat(im):
    im = np.asarray(im)
    return np.repeat(im.reshape(im.shape[0], im.shape[1], 1), 3, axis=2)


def _frame(rng, h, w, gray=False):
    im = rng.integers(0, 256, size=(h, w) if gray else (h, w, 3), dtype=np.uint8)
    im[: h // 3, : w // 4] = 255                         # a flat patch: saturated pixels in the resize
    return im


@pytest.mark.parametrize("org,net_hw", [((375, 1242), (768, 2560)), ((97, 301), (192, 640)), ((240, 320), (96, 160))])
def test_gray_array_equals_repmat(cuda, org, net_hw):
    from mscnn_b200 import ops
    rng = np.random.default_rng(org[0])
    gray = np.stack([_frame(rng, *org, gray=True) for _ in range(2)])
    want_in = np.stack([_repmat(g) for g in gray])
    pre = ops.Preprocess(org, net_hw)
    want = pre(want_in)
    for form in (gray, gray[..., None], torch.from_numpy(gray).cuda()):
        got = pre(form)
        torch.cuda.synchronize()
        assert torch.equal(got, want), type(form)


def test_gray_and_colour_mixed_list_equals_repmat(cuda):
    from mscnn_b200 import ops
    rng = np.random.default_rng(11)
    sizes = [(375, 1242), (370, 1224), (120, 400), (376, 1241), (375, 1242), (90, 300)]
    frames = [_frame(rng, h, w, gray=(i % 2 == 0)) for i, (h, w) in enumerate(sizes)]
    frames[2] = frames[2][:, :, None]                   # [h][w][1]
    want_frames = [_repmat(f) if f.ndim == 2 or f.shape[2] == 1 else f for f in frames]
    pre = ops.Preprocess(sizes[0], (768, 2560))
    want = pre(want_frames)
    got = pre(frames)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    got_dev = pre([torch.from_numpy(np.ascontiguousarray(f)).cuda() for f in frames])
    torch.cuda.synchronize()
    assert torch.equal(got_dev, want)
    # each slot equals the plan's result for that frame alone
    for n in (0, 1, 5):
        one = ops.Preprocess(sizes[n], (768, 2560))(want_frames[n][None])
        torch.cuda.synchronize()
        assert torch.equal(got[n], one[0]), n


def test_net_set_input_images_gray(cuda):
    from mscnn_b200 import models, net as mnet, ops, synth
    mnet.set_precision("fp32")
    h, w = 96, 320
    net = mnet.Net(models.kitti(h, w, 7, False, batch=3))
    net.set_params(synth.make_weights(net.layers()))
    rng = np.random.default_rng(5)
    frames = [_frame(rng, 60, 200, gray=True), _frame(rng, 75, 250), _frame(rng, 50, 170, gray=True)]
    pre = ops.Preprocess((60, 200), (h, w))
    net.set_input_images("data", pre, [_repmat(f) if f.ndim == 2 else f for f in frames])
    want = net.blob("data")
    net.set_input_images("data", pre, frames)
    assert net.blob("data").tobytes() == want.tobytes()
    arr = np.stack([_frame(rng, 60, 200, gray=True) for _ in range(3)])
    net.set_input_images("data", pre, np.stack([_repmat(a) for a in arr]))
    want = net.blob("data")
    net.set_input_images("data", pre, arr)
    assert net.blob("data").tobytes() == want.tobytes()


# ------------------------------------------------------------------------------------ (b) asynchronous pre-processing
BATCH_SIZES = [[(120, 400), (110, 380)], [(100, 320), (125, 410)], [(96, 330), (96, 330)], [(130, 420), (90, 300)],
               [(120, 400), (105, 350)]]


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


def _detect(net, cfg, classes):
    dets = torch.zeros((2, 1, cfg.max_rois_per_image, 5), device="cuda")
    cnt = torch.zeros((2, 1), dtype=torch.int32, device="cuda")
    net.detect_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    c = cnt.cpu().numpy()
    d = dets.cpu().numpy()
    return [d[i, 0, :c[i, 0]].copy() for i in range(2)]


@pytest.mark.parametrize("graph", [False, True])
def test_async_sequence_equals_sync_sequence(request, cuda, graph):
    from mscnn_b200 import capi, models, net as mnet, ops, synth
    if graph:
        request.getfixturevalue("side_stream")
    mnet.set_precision("fp32")
    h, w = 192, 640
    rng = np.random.default_rng(21)
    batches = [[_frame(rng, a, b, gray=(k == 1 and i == 0)) for i, (a, b) in enumerate(sz)]
               for k, sz in enumerate(BATCH_SIZES)]
    cfg = mnet.kitti_detect_cfg(h, w)
    classes = capi.DetectClasses.of([2])
    proto = models.kitti(h, w, 8, False, batch=2)
    ref = mnet.Net(proto)
    weights = synth.make_weights(ref.layers())
    ref.set_params(weights)
    pre_ref = ops.Preprocess((120, 400), (h, w))
    want_in, want_det = [], []
    for fr in batches:
        ref.set_input_images("data", pre_ref, fr)
        want_in.append(ref.blob("data"))
        ref.forward_only()
        want_det.append(_detect(ref, cfg, classes))
    del ref
    assert sum(len(d) for b in want_det for d in b) > 0

    net = mnet.Net(proto)
    net.set_params(weights)
    net.set_graph(graph)
    pre = ops.Preprocess((120, 400), (h, w))
    L = capi.lib()
    copy_stream = torch.cuda.ExternalStream(L.mscnn_net_copy_stream(net._h))
    net.set_input_images("data", pre, batches[0])
    assert net.blob("data").tobytes() == want_in[0].tobytes()
    replays = 0
    for k in range(len(batches)):
        net.forward_only()
        replays += int(net.graph_replayed())
        if k + 1 < len(batches):
            net.set_input_images_async("data", pre, batches[k + 1])    # while forward k is in flight
        got = _detect(net, cfg, classes)
        for i in range(2):
            assert got[i].tobytes() == want_det[k][i].tobytes(), (k, i)
        if k + 1 < len(batches):
            copy_stream.synchronize()                     # the next input has landed: read it as the next forward will
            assert net.blob("data").tobytes() == want_in[k + 1].tobytes(), k + 1
    if graph:
        assert replays >= len(batches) - 2, replays
    # the async entry does not reshape
    with pytest.raises(capi.MscnnError):
        net.set_input_images_async("data", pre, batches[0][:1])


# ------------------------------------------------------------------------------------------------ (c) the runners
DEPLOY = {"kitti_car": "kitti_car/mscnn-8s-768-trainval", "kitti_ped_cyc": "kitti_ped_cyc/mscnn-8s-768-trainval",
          "caltech": "caltech/mscnn-7s-720", "kitti_car_cascade": "kitti_car/cascade-mscnn-7s-576-2x-trainval",
          "citypersons": "citypersons/cascade-mscnn-8s-1344-2x"}
NET_HW = {"kitti_car": (192, 640), "kitti_ped_cyc": (192, 640), "caltech": (192, 256),
          "kitti_car_cascade": (192, 640), "citypersons": (336, 672)}
ORG = {"kitti_car": [(120, 400), (110, 380), (125, 410), (100, 350)],
       "caltech": [(120, 160), (100, 140), (150, 200), (90, 120)],
       "citypersons": [(160, 320), (150, 300), (200, 400), (128, 256)]}


def _deploy(name, n, h, w):
    with tarfile.open(GOLD / "deploy.tar.xz") as t:
        text = t.extractfile(f"deploy/{DEPLOY[name]}/mscnn_deploy.prototxt").read().decode()
    text, k = re.subn(r"input_dim: 1\s+input_dim: 3\s+input_dim: \d+\s+input_dim: \d+",
                      f"input_dim: {n}\ninput_dim: 3\ninput_dim: {h}\ninput_dim: {w}", text, count=1)
    assert k == 1
    return text


def _one_image_loop(net, frames, spec, net_hw):
    """The drivers' loop: one frame per forward, its ratios in the cfg (run_mscnn_detection.m:59-146,
    run_cascademscnn.m:73-146); gray frames repmat'ed first (run_cascademscnn.m:76)."""
    from mscnn_b200 import net as mnet, ops
    out = []
    for im in frames:
        im = _repmat(im) if im.ndim == 2 or im.shape[2] == 1 else im
        oh, ow = im.shape[:2]
        pre = ops.Preprocess((oh, ow), net_hw)
        net.set_input_images("data", pre, im[None])
        net.forward_only()
        cfg, classes = spec.detect_cfg(net_hw)
        ref = mnet.kitti_detect_cfg(*net_hw, org_hw=(oh, ow))
        cfg.ratio_h, cfg.ratio_w, cfg.org_h, cfg.org_w = ref.ratio_h, ref.ratio_w, ref.org_h, ref.org_w
        c = len(spec.cls_ids)
        dets = torch.zeros((1, c, cfg.max_rois_per_image, 5), device="cuda")
        cnt = torch.zeros((1, c), dtype=torch.int32, device="cuda")
        if spec.cascade:
            net.detect_cascade_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr(), stage="3rd",
                                       cls_prob=spec.blobs[1])
        else:
            net.detect_classes(cfg, classes, dets.data_ptr(), cnt.data_ptr())
        torch.cuda.synchronize()
        out.append([dets[0, s, :int(cnt[0, s])].cpu().numpy() for s in range(c)])
    return out


@pytest.mark.parametrize("name", ["kitti_car", "kitti_ped_cyc", "caltech", "kitti_car_cascade", "citypersons"])
def test_run_equals_the_one_image_loop(cuda, tmp_path, name):
    from mscnn_b200 import drivers, net as mnet, synth
    mnet.set_precision("fp32")
    spec = drivers.SPECS[name]
    net_hw = NET_HW[name]
    sizes = ORG.get(name, ORG["kitti_car"])
    rng = np.random.default_rng(len(name))
    frames = [_frame(rng, *sizes[k % len(sizes)], gray=(k % 5 == 2)) for k in range(20)]
    frames[7] = frames[7][:, :, :1] if frames[7].ndim == 3 else frames[7][:, :, None]     # [h][w][1]
    loop_net = mnet.Net(_deploy(name, 1, *net_hw))
    weights = synth.make_weights(loop_net.layers())
    loop_net.set_params(weights)
    want = _one_image_loop(loop_net, frames, spec, net_hw)
    del loop_net
    net = mnet.Net(_deploy(name, 1, *net_hw))
    net.set_params(weights)
    got = drivers.run(net, frames, spec, batch=8, net_hw=net_hw)          # batches of 8, 8 and 4
    assert len(got) == len(frames)
    assert sum(len(d) for r in want for d in r) > 0
    for i in range(len(frames)):
        assert len(got[i]) == len(spec.cls_ids)
        for s in range(len(spec.cls_ids)):
            assert got[i][s].shape == want[i][s].shape and got[i][s].tobytes() == want[i][s].tobytes(), (i, s)
    if spec.index_across_groups:              # two "cities": the index runs on across them
        a = drivers.write_results(tmp_path / "loop", spec, "c", [want[:9], want[9:]], groups=True)
        b = drivers.write_results(tmp_path / "run", spec, "c", [drivers.run(net, frames[:9], spec, net_hw=net_hw),
                                                                drivers.run(net, frames[9:], spec, net_hw=net_hw)],
                                  groups=True)
    else:
        a = drivers.write_results(tmp_path / "loop", spec, "c", want)
        b = drivers.write_results(tmp_path / "run", spec, "c", got)
    for pa, pb in zip(a, b):
        assert pa.name == pb.name and pa.read_bytes() == pb.read_bytes() and pa.stat().st_size > 0, pa.name
