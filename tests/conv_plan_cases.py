"""Runnable shapes for every pinned convolution launch plan (imported by test_conv_plan_coverage_cpu.py and
test_conv_plan_coverage_gpu.py).

A plan string (mscnn_conv_plan_describe) depends on the layer (channels, kernel, pad, stride, dilation, group, output
mode, pooling, dyn, precision and switches) and, through the pixel box, on the output extents N x Ho x Wo.  The pins of
test_conv_layout_cpu.EXPECTED and test_conv_geometry_cpu.PLAN_CASES are taken at full size; the tables here give each
pinned layer a batch and input size at which it describes to exactly its pinned string, box, stages and smem included,
so the GPU tests can run that plan and compare it with fp64:

  SMALL:    every (config, case) of EXPECTED, and every PLAN_CASES geometry (fp32-faithful, default switches), at a
            small size;
  SCHEDULE: one more size for each distinct plan string, under the config of the entry named: more than 2 x 132
            tiles (every persistent CTA of a 132-SM H100 walks at least two), a tile count that is not a multiple of 132
            (the last wave is partial), and a partial last tile in W, in H and in N wherever the box allows one (a box
            extent of 1 cannot be partial, nor can a pooled extent of 2: the pooled map's extents are even).

The layer parameters stay where they are pinned; only N, H and W are chosen here.  The entry of a row-count (dyn)
layer keeps its InnerProduct form (H = W = 1) or its 7 x 7 ROI grid.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass

from test_conv_geometry_cpu import PLAN_CASES
from test_conv_layout_cpu import BF16, CASES, CONFIGS, EXPECTED, NCHW_F32, NHWC_F32

FAKE = 0x10000       # never dereferenced: the plan query makes no CUDA call
SMS = 132            # SMs of an H100 SXM: the persistent grid of a launch with at least that many tiles
GEOMETRY_CONFIG = "fp32"


@dataclass(frozen=True)
class Layer:
    cin: int           # Cin_pad: every input channel is real
    cout: int
    cout_pad: int
    kh: int
    kw: int
    pad_h: int
    pad_w: int
    out: str           # BF16, NCHW_F32 or NHWC_F32
    pool: bool         # fused 2x2 / 2 MAX pooling
    store_full: bool   # the un-pooled planes are stored too
    dyn: bool          # a device row count
    stride: tuple = (1, 1)
    dil: tuple = (1, 1)
    group: int = 1


@dataclass(frozen=True)
class Entry:
    id: str            # "<config> <case>" (EXPECTED's key) or "fp32 <geometry case>", plus " schedule"
    key: str           # the pin's key: EXPECTED's, or "geometry <name>"
    config: str
    layer: Layer
    n: int
    h: int
    w: int
    schedule: bool

    @property
    def split(self) -> bool:
        return CONFIGS[self.config][0]

    @property
    def env(self) -> dict:
        return CONFIGS[self.config][1]


def layer_of(case: str) -> Layer:
    _, cin, _, _, cout, cout_pad, kh, kw, ph, pw, out, pool, store_full, dyn = CASES[case]
    return Layer(cin, cout, cout_pad, kh, kw, ph, pw, out, pool, store_full, dyn)


def geometry_layer(name: str) -> tuple[Layer, tuple]:
    """The PLAN_CASES layer (test_conv_geometry_cpu._desc: NHWC bf16 planes, no pooling) and its pinned full size."""
    _, args, geom, _ = next(c for c in PLAN_CASES if c[0] == name)
    n, cin, h, w, cout, kh, kw, pad = args
    ph, pw = pad if isinstance(pad, tuple) else (pad, pad)
    pad64 = lambda c: (c + 63) // 64 * 64
    layer = Layer(pad64(cin), cout, pad64(cout), kh, kw, ph, pw, BF16, False, True, False,
                  (geom.get("stride_h", 1), geom.get("stride_w", 1)), (geom.get("dil_h", 1), geom.get("dil_w", 1)),
                  geom.get("group", 1))
    return layer, (n, h, w)


def out_hw(layer: Layer, h: int, w: int) -> tuple[int, int]:
    ho = (h + 2 * layer.pad_h - (layer.dil[0] * (layer.kh - 1) + 1)) // layer.stride[0] + 1
    wo = (w + 2 * layer.pad_w - (layer.dil[1] * (layer.kw - 1) + 1)) // layer.stride[1] + 1
    return ho, wo


def desc(layer: Layer, split: bool, n: int, h: int, w: int, ptrs: dict | None = None, pool_only: bool | None = None):
    """The descriptor of one launch.  ptrs: device addresses by ConvDesc field name (x_hi, x_lo, w_hi, w_lo, bias,
    y_hi, y_lo, pool_hi, pool_lo, y_f32, dyn_n); without it every pointer the launch needs is FAKE.  pool_only: for a
    pooled layer, whether the un-pooled planes are left unstored (default: the pin's form)."""
    from mscnn_b200 import capi
    d = capi.ConvDesc()
    d.N, d.H, d.W, d.C = n, h, w, layer.cin
    d.Cout, d.Cout_pad, d.KH, d.KW, d.pad_h, d.pad_w = layer.cout, layer.cout_pad, layer.kh, layer.kw, layer.pad_h, layer.pad_w
    d.stride_h, d.stride_w = layer.stride
    d.dil_h, d.dil_w = layer.dil
    d.group = layer.group
    d.relu = int(layer.out == BF16)
    names = ["x_hi", "w_hi", "bias"] + (["x_lo", "w_lo"] if split else [])
    if layer.out == BF16:
        d.out_mode = capi.OUT_NHWC_BF16
        store = layer.store_full if pool_only is None else not pool_only
        if store or not layer.pool:
            names += ["y_hi"] + (["y_lo"] if split else [])
        if layer.pool:
            names += ["pool_hi"] + (["pool_lo"] if split else [])
    else:
        d.out_mode = capi.OUT_NCHW_F32 if layer.out == NCHW_F32 else capi.OUT_NHWC_F32
        names.append("y_f32")
    if layer.dyn:
        names.append("dyn_n")
    for k in names:
        setattr(d, k, FAKE if ptrs is None else ptrs[k])
    return d


def describe(d) -> tuple[int, str]:
    from mscnn_b200 import capi
    buf = C.create_string_buffer(512)
    rc = capi.lib().mscnn_conv_plan_describe(C.byref(d), buf, 512)
    return rc, buf.value.decode()


def box(plan: str) -> tuple[int, int, int]:
    m = re.search(r"box=(\d+)x(\d+)x(\d+)", plan)
    return int(m.group(1)), int(m.group(2)), int(m.group(3))


def n_tiles(plan: str, layer: Layer) -> int:
    block_n = int(re.search(r"conv_igemm_kernel<(\d+),", plan).group(1))
    return layer.cout_pad // block_n


def tiles(plan: str, layer: Layer, n: int, h: int, w: int) -> int:
    """Tiles of the launch (the persistent CTAs' work items): pixel boxes x BLOCK_N column tiles."""
    bw, bh, bn = box(plan)
    ho, wo = out_hw(layer, h, w)
    return -(-wo // bw) * -(-ho // bh) * -(-n // bn) * n_tiles(plan, layer)


def partial_tiles(plan: str, layer: Layer, n: int, h: int, w: int) -> dict[str, tuple[bool, bool]]:
    """Per axis: (a partial last tile is possible with this box, the size has one)."""
    bw, bh, bn = box(plan)
    ho, wo = out_hw(layer, h, w)
    step = 2 if layer.pool else 1      # pooled maps have even extents: a box of 2 always divides them
    return {"W": (bw > step, wo % bw != 0), "H": (bh > step, ho % bh != 0), "N": (bn > 1, n % bn != 0)}


# Plans whose box is as wide as the odd map it was pinned on (41 or 40 pixels): the planner picks it only where it spans
# the whole row, so their schedule entries have a partial last tile in H and N but none in W.
FULL_ROW_BOXES = {"fp32 n3_odd_w_1x1", "bf16 n3_odd_w_1x1", "fp32 n2_odd_w_nchw", "fp32_no_fat n2_odd_w_nchw",
                  "bf16 n2_odd_w_nchw", "geometry g2_128_256"}


def macs(e: Entry) -> int:
    """Multiply-adds of the fp64 reference convolution of an entry."""
    ho, wo = out_hw(e.layer, e.h, e.w)
    return e.n * ho * wo * e.layer.cout * (e.layer.cin // e.layer.group) * e.layer.kh * e.layer.kw


def pinned(key: str) -> str:
    """The pinned plan string of a key: EXPECTED's text, or a PLAN_CASES layer described at its pinned full size."""
    if key.startswith("geometry "):
        layer, (n, h, w) = geometry_layer(key.split(" ", 1)[1])
        rc, text = describe(desc(layer, True, n, h, w))
        assert rc == 0, (key, rc)
        return text
    return EXPECTED[key]


def _entry(key: str, shape: tuple, schedule: bool) -> Entry:
    n, h, w = shape
    if key.startswith("geometry "):
        layer, _ = geometry_layer(key.split(" ", 1)[1])
        config, name = GEOMETRY_CONFIG, key.split(" ", 1)[1]
    else:
        config, name = key.split(" ")
        layer = layer_of(name)
    return Entry(f"{config} {name}" + (" schedule" if schedule else ""), key, config, layer, n, h, w, schedule)


def entries() -> list[Entry]:
    return [_entry(k, s, False) for k, s in SMALL.items()] + [_entry(k, s, True) for k, s in SCHEDULE.items()]


# key: (N, H, W) -- input extents; the output extents follow from the layer's kernel, pad, stride and dilation
SMALL = {
    "fp32 conv1_2": (1, 2, 64),
    "fp32 conv2_1": (1, 1, 128),
    "fp32 conv2_2": (1, 2, 64),
    "fp32 conv3_1": (1, 1, 128),
    "fp32 conv3_2": (1, 1, 128),
    "fp32 conv3_3": (1, 2, 64),
    "fp32 conv4_1": (1, 2, 64),
    "fp32 conv4_2": (1, 2, 64),
    "fp32 conv4_3": (1, 2, 64),
    "fp32 loss1_conv1": (1, 2, 64),
    "fp32 conv5_1": (1, 4, 32),
    "fp32 conv5_3": (1, 4, 32),
    "fp32 conv6_1": (1, 8, 16),
    "fp32 LFCN_1_5x5": (1, 2, 64),
    "fp32 LFCN_1_7x7": (1, 2, 64),
    "fp32 LFCN_2_5x5": (1, 4, 32),
    "fp32 LFCN_3_7x7": (1, 8, 16),
    "fp32 LFCN_4_5x5": (4, 4, 8),
    "fp32 LFCN_4_7x7": (4, 4, 8),
    "fp32 roi_c1": (128, 7, 7),
    "fp32 fc6": (128, 1, 1),
    "fp32 cls_pred": (128, 1, 1),
    "fp32 bbox_pred": (128, 1, 1),
    "fp32 roi_c1_nchw_f32": (128, 7, 7),
    "fp32 conv1_2_pool_full": (1, 2, 64),
    "fp32 conv2_2_pool_full": (1, 2, 64),
    "fp32 conv3_3_pool_full": (1, 2, 64),
    "fp32 n1_64": (1, 2, 64),
    "fp32 n1_128_pool": (1, 4, 32),
    "fp32 n1_odd_w_64": (1, 7, 18),
    "fp32 n1_odd_w_128": (1, 7, 18),
    "fp32 n1_odd_w_256": (1, 25, 5),
    "fp32 n3_odd_w_1x1": (3, 1, 41),
    "fp32 n2_odd_w_nchw": (1, 3, 41),
    "fp32 n1_head_3x1": (1, 3, 41),
    "fp32 narrow_cout_32": (1, 8, 16),
    "fp32_no_fat conv1_2": (1, 2, 64),
    "fp32_no_fat conv2_1": (1, 1, 128),
    "fp32_no_fat conv2_2": (1, 2, 64),
    "fp32_no_fat conv3_1": (1, 1, 128),
    "fp32_no_fat conv3_2": (1, 1, 128),
    "fp32_no_fat conv3_3": (1, 2, 64),
    "fp32_no_fat conv4_1": (1, 2, 64),
    "fp32_no_fat conv4_2": (1, 2, 64),
    "fp32_no_fat conv4_3": (1, 2, 64),
    "fp32_no_fat loss1_conv1": (1, 2, 64),
    "fp32_no_fat conv5_1": (1, 4, 32),
    "fp32_no_fat conv5_3": (1, 4, 32),
    "fp32_no_fat conv6_1": (1, 8, 16),
    "fp32_no_fat LFCN_1_5x5": (1, 2, 64),
    "fp32_no_fat LFCN_1_7x7": (1, 2, 64),
    "fp32_no_fat LFCN_2_5x5": (1, 4, 32),
    "fp32_no_fat LFCN_3_7x7": (1, 8, 16),
    "fp32_no_fat LFCN_4_5x5": (4, 4, 8),
    "fp32_no_fat LFCN_4_7x7": (4, 4, 8),
    "fp32_no_fat roi_c1": (128, 7, 7),
    "fp32_no_fat fc6": (128, 1, 1),
    "fp32_no_fat cls_pred": (128, 1, 1),
    "fp32_no_fat bbox_pred": (128, 1, 1),
    "fp32_no_fat roi_c1_nchw_f32": (128, 7, 7),
    "fp32_no_fat conv1_2_pool_full": (1, 2, 64),
    "fp32_no_fat conv2_2_pool_full": (1, 2, 64),
    "fp32_no_fat conv3_3_pool_full": (1, 2, 64),
    "fp32_no_fat n1_64": (1, 2, 64),
    "fp32_no_fat n1_128_pool": (1, 4, 32),
    "fp32_no_fat n1_odd_w_64": (1, 7, 18),
    "fp32_no_fat n1_odd_w_128": (1, 7, 18),
    "fp32_no_fat n1_odd_w_256": (1, 25, 5),
    "fp32_no_fat n3_odd_w_1x1": (3, 1, 41),
    "fp32_no_fat n2_odd_w_nchw": (1, 3, 41),
    "fp32_no_fat n1_head_3x1": (1, 3, 41),
    "fp32_no_fat narrow_cout_32": (1, 8, 16),
    "fp32_no_rowshare conv1_2": (1, 2, 64),
    "fp32_no_rowshare conv2_1": (1, 1, 128),
    "fp32_no_rowshare conv2_2": (1, 2, 64),
    "fp32_no_rowshare conv3_1": (1, 1, 128),
    "fp32_no_rowshare conv3_2": (1, 1, 128),
    "fp32_no_rowshare conv3_3": (1, 2, 64),
    "fp32_no_rowshare conv4_1": (1, 2, 64),
    "fp32_no_rowshare conv4_2": (1, 2, 64),
    "fp32_no_rowshare conv4_3": (1, 2, 64),
    "fp32_no_rowshare loss1_conv1": (1, 2, 64),
    "fp32_no_rowshare conv5_1": (1, 4, 32),
    "fp32_no_rowshare conv5_3": (1, 4, 32),
    "fp32_no_rowshare conv6_1": (1, 8, 16),
    "fp32_no_rowshare LFCN_1_5x5": (1, 2, 64),
    "fp32_no_rowshare LFCN_1_7x7": (1, 2, 64),
    "fp32_no_rowshare LFCN_2_5x5": (1, 4, 32),
    "fp32_no_rowshare LFCN_3_7x7": (1, 8, 16),
    "fp32_no_rowshare LFCN_4_5x5": (4, 4, 8),
    "fp32_no_rowshare LFCN_4_7x7": (4, 4, 8),
    "fp32_no_rowshare roi_c1": (128, 7, 7),
    "fp32_no_rowshare fc6": (128, 1, 1),
    "fp32_no_rowshare cls_pred": (128, 1, 1),
    "fp32_no_rowshare bbox_pred": (128, 1, 1),
    "fp32_no_rowshare roi_c1_nchw_f32": (128, 7, 7),
    "fp32_no_rowshare conv1_2_pool_full": (1, 2, 64),
    "fp32_no_rowshare conv2_2_pool_full": (1, 2, 64),
    "fp32_no_rowshare conv3_3_pool_full": (1, 2, 64),
    "fp32_no_rowshare n1_64": (1, 2, 64),
    "fp32_no_rowshare n1_128_pool": (1, 4, 32),
    "fp32_no_rowshare n1_odd_w_64": (1, 7, 18),
    "fp32_no_rowshare n1_odd_w_128": (1, 7, 18),
    "fp32_no_rowshare n1_odd_w_256": (1, 25, 5),
    "fp32_no_rowshare n3_odd_w_1x1": (3, 1, 41),
    "fp32_no_rowshare n2_odd_w_nchw": (1, 3, 41),
    "fp32_no_rowshare n1_head_3x1": (1, 3, 41),
    "fp32_no_rowshare narrow_cout_32": (1, 8, 16),
    "bf16 conv1_2": (1, 2, 64),
    "bf16 conv2_1": (1, 1, 128),
    "bf16 conv2_2": (1, 2, 64),
    "bf16 conv3_1": (1, 1, 128),
    "bf16 conv3_2": (1, 1, 128),
    "bf16 conv3_3": (1, 2, 64),
    "bf16 conv4_1": (1, 2, 64),
    "bf16 conv4_2": (1, 2, 64),
    "bf16 conv4_3": (1, 2, 64),
    "bf16 loss1_conv1": (1, 2, 64),
    "bf16 conv5_1": (1, 4, 32),
    "bf16 conv5_3": (1, 4, 32),
    "bf16 conv6_1": (1, 8, 16),
    "bf16 LFCN_1_5x5": (1, 2, 64),
    "bf16 LFCN_1_7x7": (1, 2, 64),
    "bf16 LFCN_2_5x5": (1, 4, 32),
    "bf16 LFCN_3_7x7": (1, 8, 16),
    "bf16 LFCN_4_5x5": (4, 4, 8),
    "bf16 LFCN_4_7x7": (4, 4, 8),
    "bf16 roi_c1": (128, 7, 7),
    "bf16 fc6": (128, 1, 1),
    "bf16 cls_pred": (128, 1, 1),
    "bf16 bbox_pred": (128, 1, 1),
    "bf16 roi_c1_nchw_f32": (128, 7, 7),
    "bf16 conv1_2_pool_full": (1, 2, 64),
    "bf16 conv2_2_pool_full": (1, 2, 64),
    "bf16 conv3_3_pool_full": (1, 2, 64),
    "bf16 n1_64": (1, 2, 64),
    "bf16 n1_128_pool": (1, 4, 32),
    "bf16 n1_odd_w_64": (1, 7, 18),
    "bf16 n1_odd_w_128": (1, 7, 18),
    "bf16 n1_odd_w_256": (1, 25, 5),
    "bf16 n3_odd_w_1x1": (3, 1, 41),
    "bf16 n2_odd_w_nchw": (1, 3, 41),
    "bf16 n1_head_3x1": (1, 3, 41),
    "bf16 narrow_cout_32": (1, 8, 16),
    "bf16_no_fat conv1_2": (1, 2, 64),
    "bf16_no_fat conv2_1": (1, 1, 128),
    "bf16_no_fat conv2_2": (1, 2, 64),
    "bf16_no_fat conv3_1": (1, 1, 128),
    "bf16_no_fat conv3_2": (1, 1, 128),
    "bf16_no_fat conv3_3": (1, 2, 64),
    "bf16_no_fat conv4_1": (1, 2, 64),
    "bf16_no_fat conv4_2": (1, 2, 64),
    "bf16_no_fat conv4_3": (1, 2, 64),
    "bf16_no_fat loss1_conv1": (1, 2, 64),
    "bf16_no_fat conv5_1": (1, 4, 32),
    "bf16_no_fat conv5_3": (1, 4, 32),
    "bf16_no_fat conv6_1": (1, 8, 16),
    "bf16_no_fat LFCN_1_5x5": (1, 2, 64),
    "bf16_no_fat LFCN_1_7x7": (1, 2, 64),
    "bf16_no_fat LFCN_2_5x5": (1, 4, 32),
    "bf16_no_fat LFCN_3_7x7": (1, 8, 16),
    "bf16_no_fat LFCN_4_5x5": (4, 4, 8),
    "bf16_no_fat LFCN_4_7x7": (4, 4, 8),
    "bf16_no_fat roi_c1": (128, 7, 7),
    "bf16_no_fat fc6": (128, 1, 1),
    "bf16_no_fat cls_pred": (128, 1, 1),
    "bf16_no_fat bbox_pred": (128, 1, 1),
    "bf16_no_fat roi_c1_nchw_f32": (128, 7, 7),
    "bf16_no_fat conv1_2_pool_full": (1, 2, 64),
    "bf16_no_fat conv2_2_pool_full": (1, 2, 64),
    "bf16_no_fat conv3_3_pool_full": (1, 2, 64),
    "bf16_no_fat n1_64": (1, 2, 64),
    "bf16_no_fat n1_128_pool": (1, 4, 32),
    "bf16_no_fat n1_odd_w_64": (1, 7, 18),
    "bf16_no_fat n1_odd_w_128": (1, 7, 18),
    "bf16_no_fat n1_odd_w_256": (1, 25, 5),
    "bf16_no_fat n3_odd_w_1x1": (3, 1, 41),
    "bf16_no_fat n2_odd_w_nchw": (1, 3, 41),
    "bf16_no_fat n1_head_3x1": (1, 3, 41),
    "bf16_no_fat narrow_cout_32": (1, 8, 16),
    "bf16_no_rowshare conv1_2": (1, 2, 64),
    "bf16_no_rowshare conv2_1": (1, 1, 128),
    "bf16_no_rowshare conv2_2": (1, 2, 64),
    "bf16_no_rowshare conv3_1": (1, 1, 128),
    "bf16_no_rowshare conv3_2": (1, 1, 128),
    "bf16_no_rowshare conv3_3": (1, 2, 64),
    "bf16_no_rowshare conv4_1": (1, 2, 64),
    "bf16_no_rowshare conv4_2": (1, 2, 64),
    "bf16_no_rowshare conv4_3": (1, 2, 64),
    "bf16_no_rowshare loss1_conv1": (1, 2, 64),
    "bf16_no_rowshare conv5_1": (1, 4, 32),
    "bf16_no_rowshare conv5_3": (1, 4, 32),
    "bf16_no_rowshare conv6_1": (1, 8, 16),
    "bf16_no_rowshare LFCN_1_5x5": (1, 2, 64),
    "bf16_no_rowshare LFCN_1_7x7": (1, 2, 64),
    "bf16_no_rowshare LFCN_2_5x5": (1, 4, 32),
    "bf16_no_rowshare LFCN_3_7x7": (1, 8, 16),
    "bf16_no_rowshare LFCN_4_5x5": (4, 4, 8),
    "bf16_no_rowshare LFCN_4_7x7": (4, 4, 8),
    "bf16_no_rowshare roi_c1": (128, 7, 7),
    "bf16_no_rowshare fc6": (128, 1, 1),
    "bf16_no_rowshare cls_pred": (128, 1, 1),
    "bf16_no_rowshare bbox_pred": (128, 1, 1),
    "bf16_no_rowshare roi_c1_nchw_f32": (128, 7, 7),
    "bf16_no_rowshare conv1_2_pool_full": (1, 2, 64),
    "bf16_no_rowshare conv2_2_pool_full": (1, 2, 64),
    "bf16_no_rowshare conv3_3_pool_full": (1, 2, 64),
    "bf16_no_rowshare n1_64": (1, 2, 64),
    "bf16_no_rowshare n1_128_pool": (1, 4, 32),
    "bf16_no_rowshare n1_odd_w_64": (1, 7, 18),
    "bf16_no_rowshare n1_odd_w_128": (1, 7, 18),
    "bf16_no_rowshare n1_odd_w_256": (1, 25, 5),
    "bf16_no_rowshare n3_odd_w_1x1": (3, 1, 41),
    "bf16_no_rowshare n2_odd_w_nchw": (1, 3, 41),
    "bf16_no_rowshare n1_head_3x1": (1, 3, 41),
    "bf16_no_rowshare narrow_cout_32": (1, 8, 16),
    "geometry s2_512": (1, 7, 63),
    "geometry s4_wide": (1, 5, 253),
    "geometry s3_wide": (1, 7, 124),
    "geometry s1x2": (1, 1, 255),
    "geometry s2x1": (1, 1, 128),
    "geometry dil2": (1, 4, 32),
    "geometry dil2_w128": (1, 1, 128),
    "geometry dil2x1_w128": (1, 1, 128),
    "geometry g4_512": (1, 2, 64),
    "geometry g8_512": (1, 2, 64),
    "geometry g2_512": (1, 2, 64),
    "geometry g2_128_256": (1, 3, 40),
}

SCHEDULE = {
    "fp32 conv1_2": (7, 38, 118),
    "fp32 conv2_1": (7, 19, 251),
    "fp32 conv2_2": (7, 38, 118),
    "fp32 conv3_1": (7, 19, 251),
    "fp32 conv3_3": (7, 38, 118),
    "fp32 conv4_1": (5, 17, 187),
    "fp32 conv5_1": (3, 34, 157),
    "fp32 conv6_1": (15, 23, 45),
    "fp32 LFCN_1_5x5": (13, 13, 187),
    "fp32 LFCN_2_5x5": (13, 26, 91),
    "fp32 LFCN_3_7x7": (15, 46, 45),
    "fp32 LFCN_4_5x5": (19, 43, 37),
    "fp32 roi_c1": (763, 7, 7),
    "fp32 cls_pred": (33915, 1, 1),
    "fp32 roi_c1_nchw_f32": (763, 7, 7),
    "fp32 n1_64": (13, 13, 187),
    "fp32 n1_128_pool": (13, 26, 86),
    "fp32 n1_odd_w_64": (19, 46, 35),
    "fp32 n1_odd_w_128": (19, 46, 35),
    "fp32 n1_odd_w_256": (7, 49, 92),
    "fp32 n3_odd_w_1x1": (20, 19, 41),
    "fp32 n2_odd_w_nchw": (19, 40, 41),
    "fp32 narrow_cout_32": (15, 46, 45),
    "fp32_no_fat conv1_2": (7, 38, 118),
    "fp32_no_fat conv2_1": (7, 19, 251),
    "fp32_no_fat conv2_2": (7, 38, 118),
    "fp32_no_fat LFCN_1_5x5": (13, 13, 187),
    "fp32_no_fat LFCN_2_5x5": (13, 26, 91),
    "fp32_no_fat LFCN_3_7x7": (15, 46, 45),
    "fp32_no_fat LFCN_4_5x5": (19, 43, 37),
    "fp32_no_fat cls_pred": (33915, 1, 1),
    "fp32_no_fat n1_64": (13, 13, 187),
    "fp32_no_fat n1_128_pool": (13, 26, 86),
    "fp32_no_fat n1_odd_w_64": (19, 46, 35),
    "fp32_no_fat n1_odd_w_128": (19, 46, 35),
    "fp32_no_fat n2_odd_w_nchw": (19, 40, 41),
    "fp32_no_fat narrow_cout_32": (15, 46, 45),
    "fp32_no_rowshare conv1_2": (7, 38, 118),
    "fp32_no_rowshare conv2_1": (7, 19, 251),
    "fp32_no_rowshare conv2_2": (7, 38, 118),
    "fp32_no_rowshare n1_64": (13, 13, 187),
    "bf16 conv1_2": (7, 38, 118),
    "bf16 conv2_1": (7, 19, 251),
    "bf16 conv2_2": (7, 38, 118),
    "bf16 conv3_1": (7, 19, 251),
    "bf16 conv3_3": (7, 38, 118),
    "bf16 conv4_1": (5, 17, 187),
    "bf16 conv5_1": (3, 34, 157),
    "bf16 conv6_1": (15, 23, 45),
    "bf16 LFCN_1_5x5": (13, 13, 187),
    "bf16 LFCN_2_5x5": (13, 26, 91),
    "bf16 LFCN_3_7x7": (15, 46, 45),
    "bf16 LFCN_4_5x5": (19, 43, 37),
    "bf16 roi_c1": (763, 7, 7),
    "bf16 cls_pred": (33915, 1, 1),
    "bf16 roi_c1_nchw_f32": (763, 7, 7),
    "bf16 n1_64": (13, 13, 187),
    "bf16 n1_128_pool": (13, 26, 86),
    "bf16 n1_odd_w_64": (19, 46, 35),
    "bf16 n1_odd_w_128": (19, 46, 35),
    "bf16 n1_odd_w_256": (7, 49, 92),
    "bf16 n3_odd_w_1x1": (20, 19, 41),
    "bf16 n2_odd_w_nchw": (19, 40, 41),
    "bf16 narrow_cout_32": (15, 46, 45),
    "bf16_no_rowshare conv1_2": (7, 38, 118),
    "bf16_no_rowshare conv2_1": (7, 19, 251),
    "bf16_no_rowshare conv2_2": (7, 38, 118),
    "bf16_no_rowshare n1_64": (13, 13, 187),
    "geometry s2_512": (3, 67, 313),
    "geometry s4_wide": (1, 49, 9705),
    "geometry s3_wide": (19, 55, 241),
    "geometry s1x2": (7, 19, 501),
    "geometry s2x1": (7, 37, 251),
    "geometry dil2": (3, 34, 157),
    "geometry dil2_w128": (7, 19, 251),
    "geometry dil2x1_w128": (7, 19, 251),
    "geometry g4_512": (1, 45, 187),
    "geometry g8_512": (1, 13, 315),
    "geometry g2_512": (5, 17, 187),
    "geometry g2_128_256": (7, 55, 40),
}
