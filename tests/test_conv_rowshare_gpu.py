"""Row-share delivery of the narrow trunk convolutions (DESIGN.md 4.1c): for 3x3 layers with BLOCK_N <= 128 on 64x2 or
128x1 pixel boxes, the activation rows of a (term, dy, channel chunk) are fetched once with a one-pixel halo and serve
the three horizontal taps; only the weights are fetched per tap.  The MMAs and their order are those of the per-tap
plan (MSCNN_NO_ROWSHARE=1), so the results must be the same bit for bit.

The plan tests need no device; the others compare both deliveries on the GPU with torch.equal."""
import ctypes as C
import re

import numpy as np
import pytest


def _describe(n, cin, h, w, cout, k, pad, split=True, pooled=False, out_f32=False, dyn=False):
    from mscnn_b200 import capi
    L = capi.lib()
    d = capi.ConvDesc()
    fake = 0x10000                                   # never dereferenced: the plan query makes no CUDA call
    cpad = (cin + 63) // 64 * 64
    opad = (cout + 63) // 64 * 64
    d.x_hi, d.x_lo = fake, (fake if split else None)
    d.N, d.H, d.W, d.C = n, h, w, cpad
    d.w_hi, d.w_lo, d.bias = fake, (fake if split else None), fake
    d.Cout, d.Cout_pad, d.KH, d.KW, d.pad_h, d.pad_w = cout, opad, k, k, pad, pad
    d.relu = 1
    if out_f32:
        d.out_mode, d.y_f32 = capi.OUT_NCHW_F32, fake
    else:
        d.out_mode = capi.OUT_NHWC_BF16
        if pooled:
            d.pool_hi, d.pool_lo = fake, (fake if split else None)
        else:
            d.y_hi, d.y_lo = fake, (fake if split else None)
    if dyn:
        d.dyn_n = fake
    buf = C.create_string_buffer(512)
    rc = L.mscnn_conv_plan_describe(C.byref(d), buf, 512)
    assert rc == 0, rc
    return dict(kv.split("=", 1) for kv in re.split(r" (?=[a-z_]+=)", buf.value.decode()))


def _with_env(monkeypatch, env, fn):
    from mscnn_b200 import ops
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ops.reload_config()
    try:
        return fn()
    finally:
        for k in env:
            monkeypatch.delenv(k, raising=False)
        ops.reload_config()


# mscnn-8s-768, batch 8 (bench.py): the layers row-share serves, and the ones it must leave alone
NARROW = {"conv1_2": (8, 64, 768, 2560, 64, True), "conv2_1": (8, 64, 384, 1280, 128, False),
          "conv2_2": (8, 128, 384, 1280, 128, True)}
WIDE = {"conv3_1": (8, 128, 192, 640, 256, False), "conv3_2": (8, 256, 192, 640, 256, False),
        "conv3_3": (8, 256, 192, 640, 256, True), "conv4_1": (8, 256, 96, 320, 512, False),
        "conv4_2": (8, 512, 96, 320, 512, False), "conv5_1": (8, 512, 48, 160, 512, False),
        "conv6_1": (8, 512, 24, 80, 512, False)}


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
def test_rowshare_plans_full_size(monkeypatch, split):
    for name, (n, cin, h, w, cout, pool) in NARROW.items():
        rs = _describe(n, cin, h, w, cout, 3, 1, split=split, pooled=pool)
        per_tap = _with_env(monkeypatch, {"MSCNN_NO_ROWSHARE": "1"},
                            lambda: _describe(n, cin, h, w, cout, 3, 1, split=split, pooled=pool))
        assert rs["rowshare"] == "1" and int(rs["a_stages"]) >= 2, (name, rs)
        assert per_tap["rowshare"] == "0" and per_tap["a_stages"] == "0", (name, per_tap)
        # same instantiation and box; the weight ring (one tap per stage) at least as deep; within 227 KB
        for key in ("kernel", "box", "terms", "fat", "pool", "dyn"):
            assert rs[key] == per_tap[key], (name, key, rs, per_tap)
        assert int(rs["stages"]) >= int(per_tap["stages"]), (name, rs, per_tap)
        assert int(rs["smem"]) <= 227 * 1024, (name, rs)
    for name, (n, cin, h, w, cout, pool) in WIDE.items():
        p = _describe(n, cin, h, w, cout, 3, 1, split=split, pooled=pool)
        assert p["rowshare"] == "0" and p["a_stages"] == "0", (name, p)


def test_rowshare_plans_deeper_where_it_fits():
    p = {k: _describe(n, cin, h, w, cout, 3, 1, pooled=pool) for k, (n, cin, h, w, cout, pool) in NARROW.items()}
    assert int(p["conv1_2"]["stages"]) >= 6 and int(p["conv2_2"]["stages"]) >= 3, p
    # plain bf16: the B ring reaches its cap of 8 and the rest of the space deepens the A ring
    b = {k: _describe(n, cin, h, w, cout, 3, 1, split=False, pooled=pool) for k, (n, cin, h, w, cout, pool) in NARROW.items()}
    assert all(v["stages"] == "8" and int(v["a_stages"]) >= 3 for v in b.values()), b


def test_rowshare_not_for_heads():
    # roi_c1 (3x3 without padding on ROI rows), fc6, cls_pred, the LFCN heads (5x5 / 7x7, fp32 NCHW) and their k x 1
    # tap form (1x1 GEMM)
    plans = [_describe(16000, 1024, 7, 7, 512, 3, 0, dyn=True), _describe(16000, 12800, 1, 1, 4096, 1, 0, dyn=True),
             _describe(16000, 4096, 1, 1, 5, 1, 0, out_f32=True, dyn=True)]
    for k, pad in ((5, 2), (7, 3), (1, 0)):
        for cin, h, w in ((512, 96, 320), (512, 48, 160), (512, 24, 80), (512, 12, 40)):
            plans.append(_describe(8, cin, h, w, 9, k, pad, out_f32=True))
    for p in plans:
        assert p["rowshare"] == "0" and p["a_stages"] == "0", p


# name, N, Cin, H, W, Cout, pool, box the plan must take
CASES = [
    ("conv1_2_like",   1, 64, 8, 256, 64, True, "64x2x1"),      # 64x2, fused pool, one channel chunk
    ("conv2_2_like",   2, 128, 6, 256, 128, True, "64x2x1"),    # 64x2, fused pool, two channel chunks
    ("conv2_1_like",   2, 64, 5, 384, 128, False, "128x1x1"),   # 128x1, no pool
    ("box64x2_nopool", 1, 128, 6, 192, 64, False, "64x2x1"),    # 64x2 without pooling
    ("ragged_128x1",   1, 64, 3, 250, 128, False, "128x1x1"),   # right-edge halo past W in the zero fill
    ("ragged_64x2",    1, 128, 4, 180, 64, True, "64x2x1"),
    ("few_tiles",      1, 64, 2, 128, 64, False, "128x1x1"),    # 2 tiles: fewer tiles than SMs
    ("many_tiles",     2, 64, 64, 512, 64, True, "64x2x1"),     # many tiles per CTA through both rings
]


@pytest.mark.gpu
@pytest.mark.parametrize("no_fat", [False, True], ids=["fat", "nofat"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rowshare_bit_identical(cuda, monkeypatch, case, split, no_fat):
    import torch
    from mscnn_b200 import ops
    if no_fat and not split:
        pytest.skip("MSCNN_NO_FAT only changes the fp32-faithful plan")
    name, n, cin, h, w, cout, pool, box = case
    env = {"MSCNN_NO_FAT": "1"} if no_fat else {}
    plan = _with_env(monkeypatch, env, lambda: _describe(n, cin, h, w, cout, 3, 1, split=split, pooled=pool))
    assert plan["rowshare"] == "1" and plan["box"] == box, plan
    g = torch.Generator(device="cpu").manual_seed(1709)
    x = torch.randn((n, cin, h, w), generator=g).to(cuda)
    wt = (torch.randn((cout, cin, 3, 3), generator=g) * (2.0 / (cin * 9)) ** 0.5).to(cuda)
    b = (torch.randn((cout,), generator=g) * 0.1).to(cuda)
    xp = ops.nchw_to_planes(x, split)
    wp = ops.pack_conv_weights(wt, b, split)

    def run():
        out = ops.conv_forward(xp, wp, 1, relu=True, pool="both" if pool else None)
        torch.cuda.synchronize()
        planes = out if pool else (out,)
        return [t.clone() for pl in planes for t in (pl.hi, pl.lo) if t is not None]

    got = _with_env(monkeypatch, env, run)
    ref = _with_env(monkeypatch, {**env, "MSCNN_NO_ROWSHARE": "1"}, run)
    assert len(got) == len(ref) == (2 if split else 1) * (2 if pool else 1)
    for i, (a, r) in enumerate(zip(got, ref)):
        if not torch.equal(a, r):
            d = a != r
            pytest.fail(f"{name}: plane {i} differs in {int(d.sum())}/{d.numel()} elements, first at "
                        f"{d.nonzero()[:4].tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_rowshare_whole_net_bit_identical(cuda, monkeypatch, precision):
    """The bench net (mscnn-8s) at 192x640: every blob the same with and without row-share."""
    from mscnn_b200 import models, net as mnet, ops, synth
    mnet.set_precision(precision)
    try:
        net = mnet.Net(models.kitti(192, 640, 8, False, batch=2))
        net.set_params(synth.make_weights(net.layers()))
        net.set_input("data", synth.make_images(2, 192, 640))

        def run():
            net.forward_only()
            return {b: net.blob(b) for b in net.blob_names}

        got = run()
        ref = _with_env(monkeypatch, {"MSCNN_NO_ROWSHARE": "1"}, run)
        ops.reload_config()
    finally:
        mnet.set_precision("fp32")
    for k in ref:
        assert got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k], equal_nan=True), k
