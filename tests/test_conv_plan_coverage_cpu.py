"""The shapes of tests/conv_plan_cases.py run the pinned launch plans (no device: mscnn_conv_plan_describe only).

Every pinned (config, case) of test_conv_layout_cpu.EXPECTED and every stride / dilation / group plan of
test_conv_geometry_cpu.PLAN_CASES has a small entry that describes to exactly its pinned string, and every distinct
pinned string has a schedule entry with the tile counts and partial tiles the module states.  A new pin, a changed plan
(ring depth, box choice, staging) or a lost table row fails here and names the pin, before test_conv_plan_coverage_gpu.py
could silently run a plan other than the one pinned."""
import pytest

import conv_plan_cases as cpc
from test_conv_geometry_cpu import PLAN_CASES
from test_conv_layout_cpu import CONFIGS, EXPECTED

# Multiply-adds of all fp64 reference convolutions of test_conv_plan_coverage_gpu.py (the entries' launches, the
# pooled and head forms included once each).  About 1.2e12 today: seconds of fp64 tensor-core work on an H100, and
# the table cannot grow into a long GPU test unnoticed.
FP64_MAC_BOUND = 1.5e12

PIN_KEYS = list(EXPECTED) + [f"geometry {c[0]}" for c in PLAN_CASES]


def _set_config(config, monkeypatch):
    from mscnn_b200 import ops
    for k in ("MSCNN_NO_FAT", "MSCNN_NO_ROWSHARE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in CONFIGS[config][1].items():
        monkeypatch.setenv(k, v)
    ops.reload_config()


@pytest.fixture
def restore_config(monkeypatch):
    yield
    from mscnn_b200 import ops
    monkeypatch.undo()
    ops.reload_config()


def test_every_pin_has_an_entry():
    missing = [k for k in PIN_KEYS if k not in cpc.SMALL]
    assert not missing, f"pinned launch plans without a GPU case in conv_plan_cases.SMALL: {missing}"
    stale = [k for k in list(cpc.SMALL) + list(cpc.SCHEDULE) if k not in PIN_KEYS]
    assert not stale, f"table rows for pins that no longer exist: {stale}"


def test_every_distinct_plan_has_a_schedule_entry():
    scheduled = {cpc.pinned(k) for k in cpc.SCHEDULE}
    missing = {}
    for k in PIN_KEYS:
        plan = cpc.pinned(k)
        if plan not in scheduled:
            missing.setdefault(plan, []).append(k)
    assert not missing, "plans without a conv_plan_cases.SCHEDULE entry (pins that take them): " + "; ".join(
        f"{v} -> {p}" for p, v in missing.items())
    assert len(scheduled) == len(cpc.SCHEDULE), "two schedule entries run the same plan"


@pytest.mark.parametrize("config", list(CONFIGS))
def test_entries_describe_to_their_pins(config, monkeypatch, restore_config):
    """Also the second form of a pooled layer (pool-only vs store-both) and the run of a dyn layer without a count,
    which the GPU test launches too: the former must take the same plan, the latter the same plan but dyn=0."""
    _set_config(config, monkeypatch)
    wrong = {}
    for e in cpc.entries():
        if e.config != config:
            continue
        want = cpc.pinned(e.key)
        rc, got = cpc.describe(cpc.desc(e.layer, e.split, e.n, e.h, e.w))
        if rc != 0 or got != want:
            wrong[e.id] = (rc, got, want)
            continue
        if e.layer.pool:
            rc, other = cpc.describe(cpc.desc(e.layer, e.split, e.n, e.h, e.w, pool_only=e.layer.store_full))
            if other != want:
                wrong[e.id + " (other pooled form)"] = (rc, other, want)
        if e.layer.dyn:
            from dataclasses import replace
            rc, nodyn = cpc.describe(cpc.desc(replace(e.layer, dyn=False), e.split, e.n, e.h, e.w))
            if nodyn != want.replace("dyn=1", "dyn=0"):
                wrong[e.id + " (without a count)"] = (rc, nodyn, want)
    assert not wrong, "entries that do not run their pinned plan (rc, described, pinned): " + repr(wrong)


def test_schedule_entries_walk_many_tiles_with_partial_edges(monkeypatch, restore_config):
    bad = {}
    for e in cpc.entries():
        if not e.schedule:
            continue
        _set_config(e.config, monkeypatch)
        plan = cpc.pinned(e.key)
        t = cpc.tiles(plan, e.layer, e.n, e.h, e.w)
        if t <= 2 * cpc.SMS or t % cpc.SMS == 0:
            bad[e.id] = f"{t} tiles"
        for axis, (possible, has) in cpc.partial_tiles(plan, e.layer, e.n, e.h, e.w).items():
            if axis == "W" and e.key in cpc.FULL_ROW_BOXES:
                if cpc.box(plan)[0] != cpc.out_hw(e.layer, e.h, e.w)[1]:
                    bad[e.id] = "listed in FULL_ROW_BOXES, but its box does not span the row"
                continue
            if possible and not has:
                bad[e.id] = f"no partial last tile in {axis} (box {cpc.box(plan)}, {e.n}x{e.h}x{e.w})"
    assert not bad, bad


def test_tile_count_rule_on_a_hand_case():
    """conv1_2's plan (64x2x1 boxes, BLOCK_N 64) on 7 images of 38 x 118: ceil(118 / 64) x 38 / 2 x 7 = 266 tiles."""
    layer = cpc.layer_of("conv1_2")
    plan = EXPECTED["fp32 conv1_2"]
    assert cpc.out_hw(layer, 38, 118) == (38, 118)
    assert cpc.tiles(plan, layer, 7, 38, 118) == 266
    assert cpc.partial_tiles(plan, layer, 7, 38, 118) == {"W": (True, True), "H": (False, False), "N": (False, False)}


def test_fp64_cost_is_bounded():
    total = 0
    for e in cpc.entries():
        m = cpc.macs(e)
        total += m * (2 if e.layer.out == cpc.NHWC_F32 else 1)   # the head's gathered k x k form is checked too
    assert total <= FP64_MAC_BOUND, f"{total:.3e} fp64 multiply-adds"
