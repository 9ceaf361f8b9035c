"""The fixed-size detection drivers over the library: examples/kitti_car/run_mscnn_detection.m,
examples/kitti_ped_cyc/run_mscnn_detection.m, examples/caltech/run_mscnn_detection.m, examples/kitti_car/run_cascademscnn.m
and examples/citypersons/run_cascademscnn.m.  Each resizes every frame to one net size, runs the net, post-processes a
fixed class list and writes one dlmwrite file per class.  A spec below holds what its .m file sets, each value with the
line it comes from; `run` batches the frames and pre-processes batch k + 1 while batch k's forward runs; `write_results`
writes the drivers' files.  Every image's detections are those of the drivers' one-image-at-a-time loop, bit for bit.

    res = drivers.run(net, frames, drivers.KITTI_CAR)          # per image: [per class: [k][5] = x y w h prob]
    drivers.write_results("detections", drivers.KITTI_CAR, comp_id, res)   # detections/<comp_id>_car.txt
    res, props = drivers.run(net, frames, drivers.KITTI_CAR, proposals=True)  # + per image: float64 [k][5] proposals
    drivers.write_proposals("proposals", drivers.KITTI_CAR, comp_id, props)   # proposals/<comp_id>.txt

Several nets (make_nets: one per device entry, the weights loaded once per device and shared by the nets on it) run
the same frames with one host thread per net, each on its own stream; the result is the one-net result, bit for bit:

    nets = drivers.make_nets(proto, weights, devices=[0, 0, 1, 1])
    res = drivers.run(nets, frames, drivers.KITTI_CAR)
"""
from __future__ import annotations

import threading
from contextlib import contextmanager
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np

from . import capi

PLAIN_BLOBS = ("proposals_score", "cls_pred", "bbox_pred")   # run_mscnn_detection.m:75-77 (outputs{1..3})


@dataclass(frozen=True)
class DriverSpec:
    """What one driver script sets.  `source` maps each field to the line of the .m file that sets it."""
    script: str
    net_hw: tuple[int, int]               # imgH, imgW
    num_cls: int                          # classes of the net's cls_pred / cls_prob (bg included)
    cls_ids: tuple[int, ...]              # 1-based classes post-processed, in output order
    obj_names: tuple[str, ...] | None     # the driver's obj_names (indexed by class id), None where it has none
    cascade: bool                         # post-process of a cascade stage's decoded boxes
    blobs: tuple[str, str, str]           # the post-process's (proposals, class scores, boxes) blobs
    bbox_stds: tuple[float, ...] | None   # de-normalisation of the plain post-process; None = none (do_bb_norm = 0)
    proposal_thr: float | None            # plain post-process; None: the cascade drivers have none
    nms_overlap: float                    # pNms.overlap, type 'maxg', ovrDnm 'union'
    det_thr: float                        # <= 0: off
    result_files: tuple[str, ...]         # one per class, "{comp_id}" filled in
    index_across_groups: bool             # the image index runs across groups of frames (CityPersons' idcount)
    proposals_file: str | None = None     # the proposal list's file under proposals/, "{comp_id}" filled in; None: none
    source: dict = field(default_factory=dict, compare=False)

    def detect_cfg(self, net_hw: tuple[int, int] | None = None) -> tuple[capi.DetectCfg, capi.DetectClasses]:
        """The post-process cfg and class set at net size `net_hw` (default: the driver's own)."""
        from . import net as mnet
        h, w = net_hw or self.net_hw
        # the KITTI drivers' settings (bbox_stds [.1 .1 .2 .2], proposal_thr -10, NMS 0.5); the other drivers differ
        # only where their spec says so.  The cascade post-process reads neither bbox_stds nor proposal_thr.
        cfg = mnet.kitti_detect_cfg(h, w, num_cls=self.num_cls, cls_id=self.cls_ids[0])
        if not self.cascade:
            stds = self.bbox_stds or (1.0, 1.0, 1.0, 1.0)   # bbox_means = [], bbox_stds = []: the deltas as they are
            for k in range(4):
                cfg.bbox_std[k], cfg.bbox_mean[k] = stds[k], 0.0
            cfg.proposal_thr = self.proposal_thr
        cfg.nms_overlap = self.nms_overlap
        return cfg, capi.DetectClasses.of(self.cls_ids, self.det_thr)

    def result_paths(self, out_dir, comp_id: str) -> list[Path]:
        return [Path(out_dir) / f.format(comp_id=comp_id) for f in self.result_files]


KITTI_CAR = DriverSpec(
    script="examples/kitti_car/run_mscnn_detection.m",
    net_hw=(768, 2560), num_cls=5, cls_ids=(2,), obj_names=("bg", "car", "van", "truck", "tram"), cascade=False,
    blobs=PLAIN_BLOBS, bbox_stds=(0.1, 0.1, 0.2, 0.2), proposal_thr=-10.0, nms_overlap=0.5, det_thr=-1.0,
    result_files=("{comp_id}_car.txt",), index_across_groups=False, proposals_file="{comp_id}.txt",
    source={"net_hw": ":36", "bbox_stds": ":42-43", "nms_overlap": ":46", "cls_ids": ":48", "obj_names": ":49",
            "proposal_thr": ":51", "blobs": ":75-77", "det_thr": "none (no threshold before bbNms, :117-119)",
            "result_files": ":156-160", "index": ":150-153 (k = position in image_list)",
            "proposals": ":75-91 (keep_id :82, double then ./ ratios :86-90)",
            "proposals_file": ":162 (commented dlmwrite, index :154, cell2mat :161)",
            "num_cls": "mscnn-8s-768-trainval/mscnn_deploy.prototxt cls_pred num_output 5"})

KITTI_PED_CYC = DriverSpec(
    script="examples/kitti_ped_cyc/run_mscnn_detection.m",
    net_hw=(768, 2560), num_cls=3, cls_ids=(2, 3), obj_names=("bg", "ped", "cyc"), cascade=False,
    blobs=PLAIN_BLOBS, bbox_stds=(0.1, 0.1, 0.2, 0.2), proposal_thr=-10.0, nms_overlap=0.5, det_thr=-1.0,
    result_files=("{comp_id}_ped.txt", "{comp_id}_cyc.txt"), index_across_groups=False, proposals_file="{comp_id}.txt",
    source={"net_hw": ":36", "bbox_stds": ":42-43", "nms_overlap": ":46", "cls_ids": ":48", "obj_names": ":49",
            "proposal_thr": ":51", "blobs": ":75-77", "det_thr": "none (:117-119)", "result_files": ":156-160",
            "proposals": ":75-91 (keep_id :82, double then ./ ratios :86-90)",
            "proposals_file": ":162 (commented dlmwrite, index :154, cell2mat :161)",
            "index": ":150-153", "num_cls": "mscnn-8s-768-trainval/mscnn_deploy.prototxt cls_pred num_output 3"})

CALTECH = DriverSpec(
    script="examples/caltech/run_mscnn_detection.m",
    net_hw=(720, 960), num_cls=2, cls_ids=(2,), obj_names=("bg", "ped"), cascade=False,
    blobs=PLAIN_BLOBS, bbox_stds=None, proposal_thr=-10.0, nms_overlap=0.5, det_thr=-1.0,
    result_files=("{comp_id}_ped.txt",), index_across_groups=False, proposals_file="{comp_id}.txt",
    source={"net_hw": ":35", "bbox_stds": ":41-48 (do_bb_norm = 0: bbox_means = [], bbox_stds = [])",
            "nms_overlap": ":51", "cls_ids": ":53", "obj_names": ":54", "proposal_thr": ":56", "blobs": ":80-82",
            "det_thr": "none (:124-126)", "result_files": ":163-167", "index": ":157-160",
            "proposals": ":80-96 (keep_id :87, double then ./ ratios :91-95)",
            "proposals_file": ":169 (commented dlmwrite, index :161, cell2mat :168)",
            "num_cls": "mscnn-7s-720/mscnn_deploy.prototxt cls_pred num_output 2"})

KITTI_CAR_CASCADE = DriverSpec(
    script="examples/kitti_car/run_cascademscnn.m",
    net_hw=(576, 1920), num_cls=5, cls_ids=(2,), obj_names=("bg", "car", "van", "truck", "tram"), cascade=True,
    blobs=("proposals_3rd", "cls_prob_3rd", "output_bbox_3rd"), bbox_stds=None, proposal_thr=None, nms_overlap=0.5,
    det_thr=-1.0, result_files=("{comp_id}_car_3rd_results.txt",), index_across_groups=False,
    source={"obj_names": ":28", "cls_ids": ":29 (obj_ids)", "blobs": ":42-48 (CASCADE)", "det_thr": ":56",
            "nms_overlap": ":57", "net_hw": ":63, :79 (multiples of 32)", "gray": ":76", "result_files": ":151-157",
            "index": ":126 (kk)", "bbox_stds": "none: the net decodes the boxes (DecodeBBox)",
            "num_cls": "cascade-mscnn-7s-576-2x-trainval/mscnn_deploy.prototxt cls_prob_3rd: 5 classes"})

CITYPERSONS = DriverSpec(
    script="examples/citypersons/run_cascademscnn.m",
    net_hw=(1344, 2688), num_cls=2, cls_ids=(2,), obj_names=None, cascade=True,
    blobs=("proposals_3rd", "cls_prob_3rd_avg", "output_bbox_3rd"), bbox_stds=None, proposal_thr=None,
    nms_overlap=0.5, det_thr=-1.0, result_files=("{comp_id}_3rd_avg_results.txt",), index_across_groups=True,
    source={"cls_ids": ":31 (obj_ids)", "blobs": ":42-48 (CASCADE)", "det_thr": ":56", "nms_overlap": ":57",
            "net_hw": ":63, :85 (multiples of 32)", "gray": ":82", "result_files": ":155-165 (output_names :47)",
            "index": ":74, :131, :150 (idcount runs across the city directories :75-151)",
            "bbox_stds": "none: the net decodes the boxes (DecodeBBox)",
            "num_cls": "cascade-mscnn-8s-1344-2x/mscnn_deploy.prototxt cls_prob_3rd_avg: 2 classes"})

# The CityPersons script's default net, mscnn-8s-1344-2x-pretrained (:11): no "cascade" in its path, so CASCADE = 0
# and the script post-processes the single stage's decoded boxes.
CITYPERSONS_BASELINE = DriverSpec(
    script="examples/citypersons/run_cascademscnn.m",
    net_hw=(1344, 2688), num_cls=2, cls_ids=(2,), obj_names=None, cascade=True,
    blobs=("proposals", "cls_prob_1st", "output_bbox_1st"), bbox_stds=None, proposal_thr=None,
    nms_overlap=0.5, det_thr=-1.0, result_files=("{comp_id}_1st_results.txt",), index_across_groups=True,
    source={"script": ":11 (root_dir mscnn-8s-1344-2x-pretrained), :34-35 (CASCADE = 0)", "cls_ids": ":31 (obj_ids)",
            "obj_names": "none (the script has no obj_names)", "cascade": ":97-131 (the decoded-box post-process)",
            "blobs": ":36-41 (~CASCADE: proposals, cls_prob_1st, output_bbox_1st)", "det_thr": ":56",
            "nms_overlap": ":57", "net_hw": ":63, :85 (multiples of 32)", "gray": ":82",
            "result_files": ":155-165 (output_names {'1st'} :41)",
            "index_across_groups": ":74, :131, :150 (idcount runs across the city directories :75-151)",
            "index": ":74, :131, :150", "proposal_thr": "none: only w, h ~= 0 are filtered (:119)",
            "bbox_stds": "none: the net decodes the boxes (DecodeBBox output_bbox_1st)",
            "proposals_file": "none: the script computes no proposal list",
            "num_cls": "mscnn-8s-1344-2x/mscnn_deploy.prototxt cls_prob_1st: 2 classes"})

SPECS = {"kitti_car": KITTI_CAR, "kitti_ped_cyc": KITTI_PED_CYC, "caltech": CALTECH,
         "kitti_car_cascade": KITTI_CAR_CASCADE, "citypersons": CITYPERSONS,
         "citypersons_baseline": CITYPERSONS_BASELINE}


def make_nets(proto: str, weights, devices=(0,), reuse_activations: bool = False) -> list:
    """One net.Net of `proto` per entry of `devices` (device ids, repeats allowed), for run / widerface.run over several
    nets.  The first net on each device loads `weights` (a {layer: [blobs]} dict, as Net.set_params takes, or a
    .caffemodel path); the others on that device share its weights (Net.share_trained_layers_with), so each device
    holds one copy.  reuse_activations: each net shares one arena among the blobs whose lifetimes do not overlap
    (Net.set_activation_reuse); run and widerface.run keep the blobs their post-process reads.  The calling thread's
    device is restored."""
    import torch
    from . import net as mnet
    prev = torch.cuda.current_device()
    owners: dict[int, object] = {}
    nets = []
    try:
        for d in devices:
            mnet.set_device(int(d))
            n = mnet.Net(proto)
            if d in owners:
                n.share_trained_layers_with(owners[d])
            else:
                if isinstance(weights, dict):
                    n.set_params(weights)
                else:
                    n.copy_from(weights)
                owners[d] = n
            if reuse_activations:
                n.set_activation_reuse(True)
            nets.append(n)
    finally:
        mnet.set_device(prev)
    return nets


def keep_readable(nets, blobs) -> None:
    """Adds `blobs` to the keep set of every net of `nets` (one net or a list) that reuses activation memory, so that
    what the post-process reads after a forward is still there."""
    for n in nets if isinstance(nets, (list, tuple)) else [nets]:
        keep = getattr(n, "reuse_keep", None)
        if keep is not None and not set(blobs) <= set(keep):
            n.set_activation_reuse(True, tuple(keep) + tuple(b for b in blobs if b not in keep))


def serve_batches(nets, batches, serve) -> None:
    """Hands `batches` out whole, in order, from one queue to one host thread per net: serve(net, take) runs on its net's
    thread and calls take() for that thread's next batch, None once there are no more.  The first exception in a worker
    stops the hand-out (take() then returns None everywhere); every thread is joined before it is re-raised here."""
    if len({id(n) for n in nets}) != len(nets):
        raise ValueError("each net may appear once: one net runs on one thread")
    batches = iter(batches)
    lock = threading.Lock()
    failed: list[BaseException] = []

    def take():
        with lock:
            return None if failed else next(batches, None)

    def work(net):
        try:
            serve(net, take)
        except BaseException as e:          # noqa: BLE001 -- handed to the caller
            with lock:
                failed.append(e)

    threads = [threading.Thread(target=work, args=(n,), name=f"mscnn-net-{k}", daemon=True) for k, n in enumerate(nets)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if failed:
        raise failed[0]


@contextmanager
def net_thread(net, precision: str):
    """The calling (worker) thread set up for `net`: its device, `precision` and a stream of its own for the net and
    torch.  On exit the stream is drained and the thread's net stream reset."""
    import torch
    from . import net as mnet
    dev = net.device
    torch.cuda.set_device(dev)
    mnet.set_device(dev)
    mnet.set_precision(precision)
    stream = torch.cuda.Stream(device=dev)
    mnet.set_stream(stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            yield stream
    finally:
        stream.synchronize()
        mnet.set_stream(None)


def _plans(pre, n):
    """pre for run over n nets: None (each worker makes its own), or a list of one plan per net."""
    if pre is None:
        return [None] * n
    if not isinstance(pre, (list, tuple)) or len(pre) != n:
        raise ValueError("with several nets, pre is None or a list of one pre-processing plan per net")
    return list(pre)


def _cascade_stage(spec: DriverSpec) -> str:
    """The stage whose blobs a cascade spec reads: "1st" (proposals, output_bbox_1st) or "3rd"."""
    for stage, prop in (("1st", "proposals"), ("3rd", "proposals_3rd")):
        if spec.blobs[0] == prop and spec.blobs[2] == f"output_bbox_{stage}":
            return stage
    raise ValueError(f"unsupported cascade blobs {spec.blobs}")


def run(nets, frames, spec: DriverSpec, batch: int = 8, net_hw: tuple[int, int] | None = None, pre=None,
        proposals: bool = False):
    """Final detections of uint8 host frames ([h][w][3], or gray [h][w] / [h][w][1], any sizes) on `nets` at the one
    net size `net_hw` (default spec.net_hw), as the driver `spec` computes them.

    Returns, per image in input order, a list over spec.cls_ids of float32 [k][5] = x y w h prob in original-image
    coordinates, the kept rows in the post-process's order.  The frames run in batches of `batch` (the last one short);
    batch k + 1 is pre-processed on the net's copy stream while batch k's forward runs (Net.set_input_images_async), and
    batch k's post-process and readback follow that.  pre: an ops.Preprocess of this net size to reuse (it keeps the
    resize tables of every original size it has seen).

    nets: one net.Net, run on the calling thread and stream; or a list of nets (make_nets), each served by a host thread
    of its own on its device, in this thread's precision, on a stream of its own.  The batches are handed out whole
    in input order (serve_batches); the result is the one-net result, bit for bit.  pre is then None or one plan per
    net.

    proposals=True: returns (dets, props), props[i] being image i's proposal list, float64 [k][5] = x y w h score in
    original-image coordinates (run_mscnn_detection.m:75-91, Net.proposals), issued after the detections of the same
    batch on the same stream.  Only the plain specs have one: a cascade spec raises ValueError."""
    from . import net as mnet, ops
    if batch < 1:
        raise ValueError(f"batch ({batch}) must be positive")
    if spec.cascade:
        _cascade_stage(spec)
        if proposals:
            raise ValueError(f"{spec.script} computes no proposal list")
    frames = list(frames)
    out: list = [None] * len(frames)
    props: list | None = [None] * len(frames) if proposals else None
    if not frames:
        return (out, props) if proposals else out
    net_hw = tuple(net_hw or spec.net_hw)
    ops.image_sizes_channels(frames)                          # every frame checked before any work is issued
    keep_readable(nets, spec.blobs)
    chunks = [list(range(k, min(k + batch, len(frames)))) for k in range(0, len(frames), batch)]
    extra = (props,) if proposals else ()     # the proposal list's output, only when one is asked for
    if not isinstance(nets, (list, tuple)):
        todo = iter(chunks)
        _serve_fixed(nets, lambda: next(todo, None), frames, spec, net_hw, pre, out, *extra)
        return (out, props) if proposals else out
    plans = dict(zip(map(id, nets), _plans(pre, len(nets))))
    precision = mnet.get_precision()

    def serve(net, take):
        with net_thread(net, precision):
            _serve_fixed(net, take, frames, spec, net_hw, plans[id(net)], out, *extra)

    serve_batches(nets, chunks, serve)
    return (out, props) if proposals else out


def _serve_fixed(net, take, frames, spec: DriverSpec, net_hw, pre, out: list, props: list | None = None) -> None:
    """run's loop on one net, in the calling thread: take() gives the next batch of frame indices (None: done), and
    out[i] receives image i's detections, props[i] (props not None) its proposal list."""
    import torch
    from . import net as mnet, ops
    idx = take()
    if idx is None:
        return
    if pre is None:
        pre = ops.Preprocess(tuple(frames[0].shape[:2]), net_hw)
    elif tuple(pre.out_hw) != net_hw:
        raise ValueError(f"pre-processing plan for {pre.out_hw}, net size {net_hw}")
    cfg, classes = spec.detect_cfg(net_hw)
    c = len(spec.cls_ids)
    data = net.inputs[0]
    stream = mnet._net_stream()
    net.set_input_images(data, pre, [frames[i] for i in idx])
    while idx is not None:
        net.forward_only()
        nxt = take()
        # the same batch shape: pre-process the next batch behind this forward's first layers; a short last batch
        # reshapes the input, which waits until this batch has been post-processed
        if nxt is not None and len(nxt) == len(idx):
            net.set_input_images_async(data, pre, [frames[i] for i in nxt])
        n = len(idx)
        with torch.cuda.stream(stream):
            dets = torch.empty((n, c, cfg.max_rois_per_image, 5), dtype=torch.float32, device="cuda")
            counts = torch.empty((n, c), dtype=torch.int32, device="cuda")
            if spec.cascade:
                net.detect_cascade_classes(cfg, classes, dets.data_ptr(), counts.data_ptr(), stage=_cascade_stage(spec),
                                           cls_prob=spec.blobs[1])
            else:
                net.detect_classes(cfg, classes, dets.data_ptr(), counts.data_ptr())
            if props is not None:
                pp = read_proposals(net, cfg, n)
            cnt = counts.cpu().numpy()
            kmax = int(cnt.max()) if cnt.size else 0
            d = dets[:, :, :kmax].cpu().numpy()
        for j, i in enumerate(idx):
            out[i] = [d[j, s, :cnt[j, s]].copy() for s in range(c)]
            if props is not None:
                props[i] = pp[j]
        if nxt is not None and len(nxt) != len(idx):
            net.set_input_images(data, pre, [frames[i] for i in nxt])
        idx = nxt


def read_proposals(net, cfg, n: int) -> list[np.ndarray]:
    """Net.proposals of the last forward of `n` images, issued on the current torch stream and read back: per image
    float64 [k][5].  Only the rows up to the largest count are copied."""
    import torch
    props = torch.empty((n, cfg.max_rois_per_image, 5), dtype=torch.float64, device="cuda")
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    net.proposals(cfg, props.data_ptr(), counts.data_ptr())
    cnt = counts.cpu().numpy()
    kmax = int(cnt.max()) if cnt.size else 0
    p = props[:, :kmax].cpu().numpy()
    return [p[j, :cnt[j]].copy() for j in range(n)]


def write_proposals(out_dir, spec: DriverSpec, comp_id: str, props, first_index: int = 1) -> Path:
    """The proposal file the plain drivers leave commented out (run_mscnn_detection.m:154, :161-162;
    caltech :161, :168-169): dlmwrite(['proposals/' comp_id '.txt'], [index x y w h score]) of every image in order,
    ',' and %.5g of the float64 values (the float32 writer would round them first).  props: per image, a float64
    [k][5] list (what run(..., proposals=True) returns); image i has index first_index + i.  out_dir (created with
    its parents) plays the script's proposals/.  Returns the path written."""
    if spec.proposals_file is None:
        raise ValueError(f"{spec.script} writes no proposal list")
    path = Path(out_dir) / spec.proposals_file.format(comp_id=comp_id)
    Path(out_dir).mkdir(parents=True, exist_ok=True)
    lines = []
    for i, p in enumerate(props):
        for row in np.asarray(p, dtype=np.float64).reshape(-1, 5):
            lines.append(",".join("%.5g" % v for v in (float(first_index + i), *row.tolist())) + "\n")
    path.write_text("".join(lines))
    return path


def write_results(out_dir, spec: DriverSpec, comp_id: str, results, first_index: int = 1,
                  groups: bool = False) -> list[Path]:
    """The driver's result files under `out_dir` (created with its parents): one per class, spec.result_files, each
    the dlmwrite of [index x y w h prob] rows (',' and %.5g, kitti.write_det_file) of every image in order.

    results: per image, a list over spec.cls_ids of [k][5] rows (what `run` returns); image i has index
    first_index + i.  groups=True: a list of such lists, one per group of frames (CityPersons' city directories), the
    index running on across the groups as the driver's idcount does.  Returns the paths written."""
    from . import kitti
    images = [r for g in results for r in g] if groups else list(results)
    c = len(spec.cls_ids)
    for i, r in enumerate(images):
        if len(r) != c:
            raise ValueError(f"image {i}: {len(r)} classes, the spec has {c}")
    rows = [[np.asarray(r[s], dtype=np.float32).reshape(-1, 5) for s in range(c)] for r in images]
    paths = spec.result_paths(out_dir, comp_id)
    Path(out_dir).mkdir(parents=True, exist_ok=True)
    for s, path in enumerate(paths):
        counts = np.array([len(r[s]) for r in rows], dtype=np.int32)
        cap = max([1] + counts.tolist())
        dets = np.zeros((len(rows), cap, 5), dtype=np.float32)
        for i, r in enumerate(rows):
            dets[i, :len(r[s])] = r[s]
        kitti.write_det_file(path, dets, counts, first_image_index=first_index)
    return paths
