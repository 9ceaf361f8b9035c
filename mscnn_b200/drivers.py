"""The fixed-size detection drivers over the library: examples/kitti_car/run_mscnn_detection.m,
examples/kitti_ped_cyc/run_mscnn_detection.m, examples/caltech/run_mscnn_detection.m, examples/kitti_car/run_cascademscnn.m
and examples/citypersons/run_cascademscnn.m.  Each resizes every frame to one net size, runs the net, post-processes a
fixed class list and writes one dlmwrite file per class.  A spec below holds what its .m file sets, each value with the
line it comes from; `run` batches the frames and pre-processes batch k + 1 while batch k's forward runs; `write_results`
writes the drivers' files.  Every image's detections are those of the drivers' one-image-at-a-time loop, bit for bit.

    res = drivers.run(net, frames, drivers.KITTI_CAR)          # per image: [per class: [k][5] = x y w h prob]
    drivers.write_results("detections", drivers.KITTI_CAR, comp_id, res)   # detections/<comp_id>_car.txt
"""
from __future__ import annotations

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
    result_files=("{comp_id}_car.txt",), index_across_groups=False,
    source={"net_hw": ":36", "bbox_stds": ":42-43", "nms_overlap": ":46", "cls_ids": ":48", "obj_names": ":49",
            "proposal_thr": ":51", "blobs": ":75-77", "det_thr": "none (no threshold before bbNms, :117-119)",
            "result_files": ":156-160", "index": ":150-153 (k = position in image_list)",
            "num_cls": "mscnn-8s-768-trainval/mscnn_deploy.prototxt cls_pred num_output 5"})

KITTI_PED_CYC = DriverSpec(
    script="examples/kitti_ped_cyc/run_mscnn_detection.m",
    net_hw=(768, 2560), num_cls=3, cls_ids=(2, 3), obj_names=("bg", "ped", "cyc"), cascade=False,
    blobs=PLAIN_BLOBS, bbox_stds=(0.1, 0.1, 0.2, 0.2), proposal_thr=-10.0, nms_overlap=0.5, det_thr=-1.0,
    result_files=("{comp_id}_ped.txt", "{comp_id}_cyc.txt"), index_across_groups=False,
    source={"net_hw": ":36", "bbox_stds": ":42-43", "nms_overlap": ":46", "cls_ids": ":48", "obj_names": ":49",
            "proposal_thr": ":51", "blobs": ":75-77", "det_thr": "none (:117-119)", "result_files": ":156-160",
            "index": ":150-153", "num_cls": "mscnn-8s-768-trainval/mscnn_deploy.prototxt cls_pred num_output 3"})

CALTECH = DriverSpec(
    script="examples/caltech/run_mscnn_detection.m",
    net_hw=(720, 960), num_cls=2, cls_ids=(2,), obj_names=("bg", "ped"), cascade=False,
    blobs=PLAIN_BLOBS, bbox_stds=None, proposal_thr=-10.0, nms_overlap=0.5, det_thr=-1.0,
    result_files=("{comp_id}_ped.txt",), index_across_groups=False,
    source={"net_hw": ":35", "bbox_stds": ":41-48 (do_bb_norm = 0: bbox_means = [], bbox_stds = [])",
            "nms_overlap": ":51", "cls_ids": ":53", "obj_names": ":54", "proposal_thr": ":56", "blobs": ":80-82",
            "det_thr": "none (:124-126)", "result_files": ":163-167", "index": ":157-160",
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

SPECS = {"kitti_car": KITTI_CAR, "kitti_ped_cyc": KITTI_PED_CYC, "caltech": CALTECH,
         "kitti_car_cascade": KITTI_CAR_CASCADE, "citypersons": CITYPERSONS}


def run(net, frames, spec: DriverSpec, batch: int = 8, net_hw: tuple[int, int] | None = None, pre=None) -> list:
    """Final detections of uint8 host frames ([h][w][3], or gray [h][w] / [h][w][1], any sizes) on `net` at the one
    net size `net_hw` (default spec.net_hw), as the driver `spec` computes them.

    Returns, per image in input order, a list over spec.cls_ids of float32 [k][5] = x y w h prob in original-image
    coordinates, the kept rows in the post-process's order.  The frames run in batches of `batch` (the last one short);
    batch k + 1 is pre-processed on the net's copy stream while batch k's forward runs (Net.set_input_images_async), and
    batch k's post-process and readback follow that.  pre: an ops.Preprocess of this net size to reuse (it keeps the
    resize tables of every original size it has seen)."""
    import torch
    from . import net as mnet, ops
    if batch < 1:
        raise ValueError(f"batch ({batch}) must be positive")
    if spec.cascade and (spec.blobs[0] != "proposals_3rd" or spec.blobs[2] != "output_bbox_3rd"):
        raise ValueError(f"unsupported cascade blobs {spec.blobs}")
    frames = list(frames)
    out: list = [None] * len(frames)
    if not frames:
        return out
    net_h, net_w = net_hw or spec.net_hw
    ops.image_sizes_channels(frames)                          # every frame checked before any work is issued
    if pre is None:
        pre = ops.Preprocess(tuple(frames[0].shape[:2]), (net_h, net_w))
    elif tuple(pre.out_hw) != (net_h, net_w):
        raise ValueError(f"pre-processing plan for {pre.out_hw}, net size {(net_h, net_w)}")
    cfg, classes = spec.detect_cfg((net_h, net_w))
    c = len(spec.cls_ids)
    data = net.inputs[0]
    stream = mnet._net_stream()
    chunks = [list(range(k, min(k + batch, len(frames)))) for k in range(0, len(frames), batch)]
    net.set_input_images(data, pre, [frames[i] for i in chunks[0]])
    for k, idx in enumerate(chunks):
        net.forward_only()
        nxt = chunks[k + 1] if k + 1 < len(chunks) else None
        # the same batch shape: pre-process the next batch behind this forward's first layers; a short last batch
        # reshapes the input, which waits until this batch has been post-processed
        if nxt is not None and len(nxt) == len(idx):
            net.set_input_images_async(data, pre, [frames[i] for i in nxt])
        n = len(idx)
        with torch.cuda.stream(stream):
            dets = torch.empty((n, c, cfg.max_rois_per_image, 5), dtype=torch.float32, device="cuda")
            counts = torch.empty((n, c), dtype=torch.int32, device="cuda")
            if spec.cascade:
                net.detect_cascade_classes(cfg, classes, dets.data_ptr(), counts.data_ptr(), stage="3rd",
                                           cls_prob=spec.blobs[1])
            else:
                net.detect_classes(cfg, classes, dets.data_ptr(), counts.data_ptr())
            cnt = counts.cpu().numpy()
            kmax = int(cnt.max()) if cnt.size else 0
            d = dets[:, :, :kmax].cpu().numpy()
        for j, i in enumerate(idx):
            out[i] = [d[j, s, :cnt[j, s]].copy() for s in range(c)]
        if nxt is not None and len(nxt) != len(idx):
            net.set_input_images(data, pre, [frames[i] for i in nxt])
    return out


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
