"""The activation memory plan (Net::set_activation_reuse), host only: nets are built without a device, as in
test_net_cpu.py, and the plan is made from their structure and shapes without allocating anything.

(a) For all 23 shipped deploy nets, at their drivers' net sizes, batch 8, both precisions: no two storages that are
    live at the same layer share arena bytes, every offset is 256-byte aligned, inputs / outputs / kept blobs are
    outside the arena, and the arena is smaller than what the planned storages take without reuse.
(b) The plan of mscnn-8s-768 at 8 x 768 x 2560 is pinned in both precisions, and at an odd extent where the folded
    pools run themselves (the un-pooled convolution tops then take bytes).
(c) The refusals: a keep name that is not a blob, a partial forward over a planned blob written before it.
(d) A net with reuse off reports no plan."""
import hashlib
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
DEPLOY_ARCHIVE = ROOT / "tests" / "golden" / "deploy.tar.xz"
LINE = re.compile(r"^(\S+) (\d+) (\d+)-(\d+) (@(\d+)|input|output|kept)$")


@pytest.fixture(scope="module")
def REF_EX(tmp_path_factory):
    import tarfile
    d = tmp_path_factory.mktemp("deploy")
    with tarfile.open(DEPLOY_ARCHIVE) as t:
        t.extractall(d, filter="data")
    return d / "deploy"


@pytest.fixture()
def precision():
    from mscnn_b200 import net as mnet
    prev = mnet.get_precision()
    yield mnet.set_precision
    mnet.set_precision(prev)


def _net_hw(rel: str) -> tuple[int, int]:
    """The net size the dataset's driver runs the model at (drivers.SPECS; WIDER: one of its bucketed sizes)."""
    from mscnn_b200 import drivers
    dataset, model = rel.split("/")
    if dataset == "widerface":
        return (1024, 768)
    if dataset == "kitti_car" and model.startswith("cascade"):
        return drivers.KITTI_CAR_CASCADE.net_hw
    return {"kitti_car": drivers.KITTI_CAR, "kitti_ped_cyc": drivers.KITTI_PED_CYC, "caltech": drivers.CALTECH,
            "citypersons": drivers.CITYPERSONS}[dataset].net_hw


def _sized(net, n, h, w):
    net.reshape_input("data", n, 3, h, w)
    return net


def _parse(text):
    rows = []
    for line in text.splitlines():
        m = LINE.match(line)
        assert m, line
        rows.append(dict(blob=m[1], bytes=int(m[2]), first=int(m[3]), last=int(m[4]),
                         offset=int(m[6]) if m[6] else None, outside=None if m[6] else m[5]))
    return rows


def _check_plan(net, keep):
    arena, without = net.activation_bytes()
    rows = _parse(net.activation_plan())
    planned = [r for r in rows if r["offset"] is not None]
    assert planned and 0 < arena < without
    assert sum(r["bytes"] for r in planned) == without
    for r in planned:
        assert r["offset"] % 256 == 0 and r["bytes"] % 256 == 0
        assert r["offset"] + r["bytes"] <= arena
        assert r["blob"] not in net.inputs and r["blob"] not in net.outputs and r["blob"] not in keep
    for a_i, a in enumerate(planned):
        for b in planned[a_i + 1:]:
            live_together = a["first"] <= b["last"] and b["first"] <= a["last"]
            if live_together:
                assert a["offset"] + a["bytes"] <= b["offset"] or b["offset"] + b["bytes"] <= a["offset"], (a, b)
    outside = {r["blob"]: r["outside"] for r in rows if r["offset"] is None}
    for b in net.inputs:
        assert outside[b] == "input"
    for b in keep:
        assert outside.get(b) in ("kept", "output", "input"), b
    for b in net.outputs:
        if b in outside:
            assert outside[b] in ("output", "input")
    return arena, without


def test_every_shipped_net_plans_without_overlap(REF_EX, precision):
    from mscnn_b200.net import Net
    files = sorted(REF_EX.glob("*/*/mscnn_deploy.prototxt"))
    assert len(files) == 23
    for f in files:
        rel = str(f.parent.relative_to(REF_EX))
        net = _sized(Net(str(f)), 8, *_net_hw(rel))
        keep = ("conv4_3",) if "conv4_3" in net.blob_names else ()
        net.set_activation_reuse(True, keep)
        sizes = {}
        for mode in ("fp32", "bf16"):
            precision(mode)
            sizes[mode] = _check_plan(net, keep)
        # the lo planes only exist in fp32-faithful precision
        assert sizes["bf16"][1] < sizes["fp32"][1], rel


# mscnn-8s-768 at batch 8: (arena bytes, bytes without reuse, sha256 of the describe text)
PINNED = {
    ("fp32", 768, 2560): (5033164800, 16718461440, "a5fc6f4fc0c21cd1719175f5b1376c50bce89ce2fdc4e8c14c50080693857f6c"),
    ("bf16", 768, 2560): (2516582400, 8371141120, "466b4bccdfea52f19ab3795a887cfbdba3d7cc8751a104d34c9cabc6db5266a1"),
    ("fp32", 769, 2561): (8066699264, 23868664832, "0f2e71033912a7f63f0ba09534d748385a295f0d15f955c51f7ae8a65def3265"),
    ("bf16", 769, 2561): (4033349632, 11946469376, "17a5dfe2d4620db6a1e64108d5d084bdb0165af9c0993d529a72cc29a5e5cc7f"),
}


@pytest.mark.parametrize("mode,h,w", sorted(PINNED))
def test_kitti_8s_plan_is_pinned(REF_EX, precision, mode, h, w):
    from mscnn_b200.net import Net
    net = _sized(Net(str(REF_EX / "kitti_car/mscnn-8s-768-trainval/mscnn_deploy.prototxt")), 8, h, w)
    net.set_activation_reuse(True)
    precision(mode)
    text = net.activation_plan()
    arena, without = _check_plan(net, ())
    got = (arena, without, hashlib.sha256(text.encode()).hexdigest())
    assert got == PINNED[(mode, h, w)], text
    rows = {r["blob"]: r for r in _parse(text)}
    if h % 2:
        # odd extents: conv1_2 stores its full top and pool1 runs itself, one layer later
        assert rows["conv1_2"]["bytes"] > 0 and rows["pool1"]["first"] == rows["conv1_2"]["last"]
    else:
        assert "conv1_2" not in rows                      # pooled in conv1_2's epilogue: the full top takes no bytes
        assert rows["pool1"]["first"] == rows["conv1_1"]["last"]
    # the blobs behind BoxOutput are planned at the cap row count (8 images x max_nms_num)
    assert rows["proposals"]["bytes"] >= 8 * 2000 * 5 * 4


def test_keep_name_that_is_not_a_blob_is_refused():
    from mscnn_b200 import capi, models
    from mscnn_b200.net import Net
    net = Net(models.kitti(384, 1280))
    with pytest.raises(capi.MscnnError, match="Cannot keep 'conv9_9' readable under activation reuse: net '.*' has no "
                                              "blob of that name"):
        net.set_activation_reuse(True, ["conv4_3", "conv9_9"])
    assert net.reuse_keep is None and net.activation_bytes() == (0, 0)


def test_partial_forward_over_an_unkept_blob_is_refused():
    from mscnn_b200 import capi, models
    from mscnn_b200.net import Net
    net = Net(models.kitti(384, 1280))
    net.set_activation_reuse(True, ["conv4_3"])     # the ROI head's feature map is kept, the first proposal map is not
    with pytest.raises(capi.MscnnError, match="ForwardFromTo\\(\\d+, \\d+\\) with activation reuse on: layer 'proposals' "
                                              "reads blob 'LFCN_1_5x5', which is written before layer 'conv5_1' and whose "
                                              "storage other blobs reuse; keep it"):
        net.forward_only(start="conv5_1")


def test_reuse_off_reports_no_plan():
    from mscnn_b200 import models
    from mscnn_b200.net import Net
    net = Net(models.kitti(384, 1280))
    assert net.activation_bytes() == (0, 0) and net.activation_plan() == ""
    net.set_activation_reuse(True)
    assert net.activation_bytes()[0] > 0
    net.set_activation_reuse(False)
    assert net.activation_bytes() == (0, 0) and net.activation_plan() == "" and net.reuse_keep is None
