"""The complete launch plan (mscnn_conv_plan_describe) of every convolution and InnerProduct of the bench net and of
the shapes the other tests reach, in fp32-faithful and plain bf16, each also under MSCNN_NO_FAT=1 and
MSCNN_NO_ROWSHARE=1.  The `smem=` field is the shared memory the launch reserves, computed by the same layout function
the kernel carves its regions with; these strings pin it, the ring depths and the staging buffers byte for byte."""
import ctypes as C

import pytest

FAKE = 0x10000   # never dereferenced: the plan query makes no CUDA call
BF16, NCHW_F32, NHWC_F32 = "bf16", "nchw_f32", "nhwc_f32"

# name: (N, Cin_pad, H, W, Cout, Cout_pad, KH, KW, pad_h, pad_w, out, pool, store_full, dyn)
#   pool: fused 2x2 MAX pooling of the output; store_full: the un-pooled output is stored too (y_hi set)
CASES = {
    # mscnn-8s, batch 8, 3x768x2560 (the bench net); conv1_1 has its own kernel
    "conv1_2": (8, 64, 768, 2560, 64, 64, 3, 3, 1, 1, BF16, True, False, False),
    "conv2_1": (8, 64, 384, 1280, 128, 128, 3, 3, 1, 1, BF16, False, True, False),
    "conv2_2": (8, 128, 384, 1280, 128, 128, 3, 3, 1, 1, BF16, True, False, False),
    "conv3_1": (8, 128, 192, 640, 256, 256, 3, 3, 1, 1, BF16, False, True, False),
    "conv3_2": (8, 256, 192, 640, 256, 256, 3, 3, 1, 1, BF16, False, True, False),
    "conv3_3": (8, 256, 192, 640, 256, 256, 3, 3, 1, 1, BF16, True, False, False),
    "conv4_1": (8, 256, 96, 320, 512, 512, 3, 3, 1, 1, BF16, False, True, False),
    "conv4_2": (8, 512, 96, 320, 512, 512, 3, 3, 1, 1, BF16, False, True, False),
    "conv4_3": (8, 512, 96, 320, 512, 512, 3, 3, 1, 1, BF16, False, True, False),
    "loss1_conv1": (8, 512, 96, 320, 512, 512, 3, 3, 1, 1, BF16, False, True, False),
    "conv5_1": (8, 512, 48, 160, 512, 512, 3, 3, 1, 1, BF16, False, True, False),
    "conv5_3": (8, 512, 48, 160, 512, 512, 3, 3, 1, 1, BF16, False, True, False),
    "conv6_1": (8, 512, 24, 80, 512, 512, 3, 3, 1, 1, BF16, False, True, False),
    # LFCN k x k heads as k x 1 convolutions with k * 9 columns (pixel-major fp32 partial sums)
    "LFCN_1_5x5": (8, 512, 96, 320, 64, 64, 5, 1, 2, 0, NHWC_F32, False, False, False),
    "LFCN_1_7x7": (8, 512, 96, 320, 64, 64, 7, 1, 3, 0, NHWC_F32, False, False, False),
    "LFCN_2_5x5": (8, 512, 48, 160, 64, 64, 5, 1, 2, 0, NHWC_F32, False, False, False),
    "LFCN_3_7x7": (8, 512, 24, 80, 64, 64, 7, 1, 3, 0, NHWC_F32, False, False, False),
    "LFCN_4_5x5": (8, 512, 12, 40, 64, 64, 5, 1, 2, 0, NHWC_F32, False, False, False),
    "LFCN_4_7x7": (8, 512, 12, 40, 64, 64, 7, 1, 3, 0, NHWC_F32, False, False, False),
    # ROI head with a device row count
    "roi_c1": (16000, 1024, 7, 7, 512, 512, 3, 3, 0, 0, BF16, False, True, True),
    "fc6": (16000, 12800, 1, 1, 4096, 4096, 1, 1, 0, 0, BF16, False, True, True),
    "cls_pred": (16000, 4096, 1, 1, 5, 64, 1, 1, 0, 0, NCHW_F32, False, False, True),
    "bbox_pred": (16000, 4096, 1, 1, 20, 64, 1, 1, 0, 0, NCHW_F32, False, False, True),
    "roi_c1_nchw_f32": (16000, 1024, 7, 7, 512, 512, 3, 3, 0, 0, NCHW_F32, False, False, True),
    # pooled with the un-pooled output stored too
    "conv1_2_pool_full": (8, 64, 768, 2560, 64, 64, 3, 3, 1, 1, BF16, True, True, False),
    "conv2_2_pool_full": (8, 128, 384, 1280, 128, 128, 3, 3, 1, 1, BF16, True, True, False),
    "conv3_3_pool_full": (8, 256, 192, 640, 256, 256, 3, 3, 1, 1, BF16, True, True, False),
    # one image, odd widths, small maps
    "n1_64": (1, 64, 96, 320, 64, 64, 3, 3, 1, 1, BF16, False, True, False),
    "n1_128_pool": (1, 128, 48, 160, 128, 128, 3, 3, 1, 1, BF16, True, False, False),
    "n1_odd_w_64": (1, 64, 97, 321, 64, 64, 3, 3, 1, 1, BF16, False, True, False),
    "n1_odd_w_128": (1, 128, 49, 161, 128, 128, 3, 3, 1, 1, BF16, False, True, False),
    "n1_odd_w_256": (1, 256, 25, 81, 256, 256, 3, 3, 1, 1, BF16, False, True, False),
    "n3_odd_w_1x1": (3, 512, 13, 41, 512, 512, 1, 1, 0, 0, BF16, False, True, False),
    "n2_odd_w_nchw": (2, 512, 13, 41, 9, 64, 3, 3, 1, 1, NCHW_F32, False, False, False),
    "n1_head_3x1": (1, 512, 12, 41, 27, 64, 3, 1, 1, 0, NHWC_F32, False, False, False),
    "narrow_cout_32": (2, 64, 24, 80, 20, 32, 3, 3, 1, 1, NCHW_F32, False, False, False),
}
CONFIGS = {
    "fp32": (True, {}), "fp32_no_fat": (True, {"MSCNN_NO_FAT": "1"}),
    "fp32_no_rowshare": (True, {"MSCNN_NO_ROWSHARE": "1"}),
    "bf16": (False, {}), "bf16_no_fat": (False, {"MSCNN_NO_FAT": "1"}),
    "bf16_no_rowshare": (False, {"MSCNN_NO_ROWSHARE": "1"}),
}


def plan(case: str, split: bool) -> str:
    from mscnn_b200 import capi
    n, cin, h, w, cout, cout_pad, kh, kw, ph, pw, out, pool, store_full, dyn = CASES[case]
    d = capi.ConvDesc()
    d.x_hi, d.x_lo = FAKE, (FAKE if split else None)
    d.N, d.H, d.W, d.C = n, h, w, cin
    d.w_hi, d.w_lo, d.bias = FAKE, (FAKE if split else None), FAKE
    d.Cout, d.Cout_pad, d.KH, d.KW, d.pad_h, d.pad_w = cout, cout_pad, kh, kw, ph, pw
    d.relu = int(out == BF16)
    if out == BF16:
        d.out_mode = capi.OUT_NHWC_BF16
        if store_full:
            d.y_hi, d.y_lo = FAKE, (FAKE if split else None)
        if pool:
            d.pool_hi, d.pool_lo = FAKE, (FAKE if split else None)
    else:
        d.out_mode, d.y_f32 = (capi.OUT_NCHW_F32 if out == NCHW_F32 else capi.OUT_NHWC_F32), FAKE
    if dyn:
        d.dyn_n = FAKE
    buf = C.create_string_buffer(512)
    rc = capi.lib().mscnn_conv_plan_describe(C.byref(d), buf, 512)
    assert rc == 0, (case, rc)
    return buf.value.decode()


def plans(config: str, monkeypatch) -> dict[str, str]:
    from mscnn_b200 import ops
    split, env = CONFIGS[config]
    for k in ("MSCNN_NO_FAT", "MSCNN_NO_ROWSHARE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ops.reload_config()
    try:
        return {case: plan(case, split) for case in CASES}
    finally:
        monkeypatch.undo()
        ops.reload_config()


@pytest.mark.parametrize("config", list(CONFIGS))
def test_plan_strings_are_pinned(config, monkeypatch):
    got = plans(config, monkeypatch)
    want = {case: EXPECTED[f"{config} {case}"] for case in CASES}
    diff = {case: (got[case], want[case]) for case in CASES if got[case] != want[case]}
    assert not diff, diff


# A change to any of these is a change of launch plan, not a refactor.
EXPECTED = {
    "fp32 conv1_2":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=1 stages=7 epi_bufs=1 smem=226496 dyn=0 rowshare=1 a_stages=2",
    "fp32 conv2_1":
        "kernel=conv_igemm_kernel<128, true> box=128x1x1 terms=3 fat=1 pool=0 stages=3 epi_bufs=1 smem=201920 dyn=0 rowshare=1 a_stages=2",
    "fp32 conv2_2":
        "kernel=conv_igemm_kernel<128, true> box=64x2x1 terms=3 fat=1 pool=1 stages=3 epi_bufs=1 smem=210112 dyn=0 rowshare=1 a_stages=2",
    "fp32 conv3_1":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv3_2":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv3_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv4_1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv4_2":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv4_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 loss1_conv1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv5_1":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv5_3":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 conv6_1":
        "kernel=conv_igemm_kernel<256, false> box=16x8x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 LFCN_1_5x5":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 LFCN_1_7x7":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 LFCN_2_5x5":
        "kernel=conv_igemm_kernel<64, true> box=32x4x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 LFCN_3_7x7":
        "kernel=conv_igemm_kernel<64, true> box=16x8x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 LFCN_4_5x5":
        "kernel=conv_igemm_kernel<64, true> box=8x4x4 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 LFCN_4_7x7":
        "kernel=conv_igemm_kernel<64, true> box=8x4x4 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 roi_c1":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "fp32 fc6":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "fp32 cls_pred":
        "kernel=conv_igemm_kernel<64, true> box=1x1x128 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32 bbox_pred":
        "kernel=conv_igemm_kernel<64, true> box=1x1x128 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32 roi_c1_nchw_f32":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32 conv1_2_pool_full":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=1 stages=7 epi_bufs=1 smem=226496 dyn=0 rowshare=1 a_stages=2",
    "fp32 conv2_2_pool_full":
        "kernel=conv_igemm_kernel<128, true> box=64x2x1 terms=3 fat=1 pool=1 stages=3 epi_bufs=1 smem=210112 dyn=0 rowshare=1 a_stages=2",
    "fp32 conv3_3_pool_full":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32 n1_64":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=0 stages=7 epi_bufs=1 smem=218304 dyn=0 rowshare=1 a_stages=2",
    "fp32 n1_128_pool":
        "kernel=conv_igemm_kernel<128, true> box=32x4x1 terms=3 fat=1 pool=1 stages=2 epi_bufs=1 smem=173184 dyn=0 rowshare=0 a_stages=0",
    "fp32 n1_odd_w_64":
        "kernel=conv_igemm_kernel<64, true> box=18x7x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 n1_odd_w_128":
        "kernel=conv_igemm_kernel<128, true> box=18x7x1 terms=3 fat=1 pool=0 stages=3 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 n1_odd_w_256":
        "kernel=conv_igemm_kernel<256, false> box=5x25x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 n3_odd_w_1x1":
        "kernel=conv_igemm_kernel<256, false> box=41x1x3 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32 n2_odd_w_nchw":
        "kernel=conv_igemm_kernel<64, true> box=41x3x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 n1_head_3x1":
        "kernel=conv_igemm_kernel<64, true> box=41x3x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32 narrow_cout_32":
        "kernel=conv_igemm_kernel<32, true> box=16x8x1 terms=3 fat=1 pool=0 stages=5 epi_bufs=0 smem=205952 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv1_2":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=3 fat=0 pool=1 stages=8 epi_bufs=1 smem=177344 dyn=0 rowshare=1 a_stages=4",
    "fp32_no_fat conv2_1":
        "kernel=conv_igemm_kernel<128, false> box=128x1x1 terms=3 fat=0 pool=0 stages=7 epi_bufs=2 smem=216256 dyn=0 rowshare=1 a_stages=2",
    "fp32_no_fat conv2_2":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=3 fat=0 pool=1 stages=6 epi_bufs=2 smem=216256 dyn=0 rowshare=1 a_stages=2",
    "fp32_no_fat conv3_1":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv3_2":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv3_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv4_1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv4_2":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv4_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat loss1_conv1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv5_1":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv5_3":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat conv6_1":
        "kernel=conv_igemm_kernel<256, false> box=16x8x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat LFCN_1_5x5":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat LFCN_1_7x7":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat LFCN_2_5x5":
        "kernel=conv_igemm_kernel<64, false> box=32x4x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat LFCN_3_7x7":
        "kernel=conv_igemm_kernel<64, false> box=16x8x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat LFCN_4_5x5":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat LFCN_4_7x7":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat roi_c1":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_fat fc6":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_fat cls_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_fat bbox_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_fat roi_c1_nchw_f32":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_fat conv1_2_pool_full":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=3 fat=0 pool=1 stages=8 epi_bufs=1 smem=177344 dyn=0 rowshare=1 a_stages=4",
    "fp32_no_fat conv2_2_pool_full":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=3 fat=0 pool=1 stages=6 epi_bufs=2 smem=216256 dyn=0 rowshare=1 a_stages=2",
    "fp32_no_fat conv3_3_pool_full":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat n1_64":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=1 smem=169152 dyn=0 rowshare=1 a_stages=4",
    "fp32_no_fat n1_128_pool":
        "kernel=conv_igemm_kernel<128, false> box=32x4x1 terms=3 fat=0 pool=1 stages=4 epi_bufs=2 smem=214144 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat n1_odd_w_64":
        "kernel=conv_igemm_kernel<64, false> box=18x7x1 terms=3 fat=0 pool=0 stages=6 epi_bufs=2 smem=214144 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat n1_odd_w_128":
        "kernel=conv_igemm_kernel<128, false> box=18x7x1 terms=3 fat=0 pool=0 stages=5 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat n1_odd_w_256":
        "kernel=conv_igemm_kernel<256, false> box=5x25x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat n3_odd_w_1x1":
        "kernel=conv_igemm_kernel<256, false> box=41x1x3 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat n2_odd_w_nchw":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat n1_head_3x1":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_fat narrow_cout_32":
        "kernel=conv_igemm_kernel<32, false> box=16x8x1 terms=3 fat=0 pool=0 stages=8 epi_bufs=0 smem=164992 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv1_2":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv2_1":
        "kernel=conv_igemm_kernel<128, true> box=128x1x1 terms=3 fat=1 pool=0 stages=3 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv2_2":
        "kernel=conv_igemm_kernel<128, true> box=64x2x1 terms=3 fat=1 pool=1 stages=2 epi_bufs=1 smem=173184 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv3_1":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv3_2":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv3_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv4_1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv4_2":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv4_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare loss1_conv1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv5_1":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv5_3":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv6_1":
        "kernel=conv_igemm_kernel<256, false> box=16x8x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare LFCN_1_5x5":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare LFCN_1_7x7":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare LFCN_2_5x5":
        "kernel=conv_igemm_kernel<64, true> box=32x4x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare LFCN_3_7x7":
        "kernel=conv_igemm_kernel<64, true> box=16x8x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare LFCN_4_5x5":
        "kernel=conv_igemm_kernel<64, true> box=8x4x4 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare LFCN_4_7x7":
        "kernel=conv_igemm_kernel<64, true> box=8x4x4 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare roi_c1":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_rowshare fc6":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_rowshare cls_pred":
        "kernel=conv_igemm_kernel<64, true> box=1x1x128 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_rowshare bbox_pred":
        "kernel=conv_igemm_kernel<64, true> box=1x1x128 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_rowshare roi_c1_nchw_f32":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=3 fat=0 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv1_2_pool_full":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv2_2_pool_full":
        "kernel=conv_igemm_kernel<128, true> box=64x2x1 terms=3 fat=1 pool=1 stages=2 epi_bufs=1 smem=173184 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare conv3_3_pool_full":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=3 fat=0 pool=1 stages=3 epi_bufs=1 smem=189568 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n1_64":
        "kernel=conv_igemm_kernel<64, true> box=64x2x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n1_128_pool":
        "kernel=conv_igemm_kernel<128, true> box=32x4x1 terms=3 fat=1 pool=1 stages=2 epi_bufs=1 smem=173184 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n1_odd_w_64":
        "kernel=conv_igemm_kernel<64, true> box=18x7x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n1_odd_w_128":
        "kernel=conv_igemm_kernel<128, true> box=18x7x1 terms=3 fat=1 pool=0 stages=3 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n1_odd_w_256":
        "kernel=conv_igemm_kernel<256, false> box=5x25x1 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n3_odd_w_1x1":
        "kernel=conv_igemm_kernel<256, false> box=41x1x3 terms=3 fat=0 pool=0 stages=4 epi_bufs=1 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n2_odd_w_nchw":
        "kernel=conv_igemm_kernel<64, true> box=41x3x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare n1_head_3x1":
        "kernel=conv_igemm_kernel<64, true> box=41x3x1 terms=3 fat=1 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "fp32_no_rowshare narrow_cout_32":
        "kernel=conv_igemm_kernel<32, true> box=16x8x1 terms=3 fat=1 pool=0 stages=5 epi_bufs=0 smem=205952 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv1_2":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=1 smem=156864 dyn=0 rowshare=1 a_stages=4",
    "bf16 conv2_1":
        "kernel=conv_igemm_kernel<128, false> box=128x1x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=2 smem=217280 dyn=0 rowshare=1 a_stages=3",
    "bf16 conv2_2":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=2 smem=225472 dyn=0 rowshare=1 a_stages=3",
    "bf16 conv3_1":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv3_2":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv3_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=1 stages=4 epi_bufs=1 smem=218240 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv4_1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv4_2":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv4_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 loss1_conv1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv5_1":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv5_3":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 conv6_1":
        "kernel=conv_igemm_kernel<256, false> box=16x8x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 LFCN_1_5x5":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 LFCN_1_7x7":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 LFCN_2_5x5":
        "kernel=conv_igemm_kernel<64, false> box=32x4x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 LFCN_3_7x7":
        "kernel=conv_igemm_kernel<64, false> box=16x8x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 LFCN_4_5x5":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 LFCN_4_7x7":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 roi_c1":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "bf16 fc6":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "bf16 cls_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16 bbox_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16 roi_c1_nchw_f32":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16 conv1_2_pool_full":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=1 smem=156864 dyn=0 rowshare=1 a_stages=4",
    "bf16 conv2_2_pool_full":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=2 smem=225472 dyn=0 rowshare=1 a_stages=3",
    "bf16 conv3_3_pool_full":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=1 stages=4 epi_bufs=1 smem=218240 dyn=0 rowshare=0 a_stages=0",
    "bf16 n1_64":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=1 smem=152768 dyn=0 rowshare=1 a_stages=4",
    "bf16 n1_128_pool":
        "kernel=conv_igemm_kernel<128, false> box=32x4x1 terms=1 fat=0 pool=1 stages=5 epi_bufs=2 smem=205952 dyn=0 rowshare=0 a_stages=0",
    "bf16 n1_odd_w_64":
        "kernel=conv_igemm_kernel<64, false> box=18x7x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 n1_odd_w_128":
        "kernel=conv_igemm_kernel<128, false> box=18x7x1 terms=1 fat=0 pool=0 stages=6 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 n1_odd_w_256":
        "kernel=conv_igemm_kernel<256, false> box=5x25x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 n3_odd_w_1x1":
        "kernel=conv_igemm_kernel<256, false> box=41x1x3 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16 n2_odd_w_nchw":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 n1_head_3x1":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16 narrow_cout_32":
        "kernel=conv_igemm_kernel<32, false> box=16x8x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=164992 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv1_2":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=1 smem=156864 dyn=0 rowshare=1 a_stages=4",
    "bf16_no_fat conv2_1":
        "kernel=conv_igemm_kernel<128, false> box=128x1x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=2 smem=217280 dyn=0 rowshare=1 a_stages=3",
    "bf16_no_fat conv2_2":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=2 smem=225472 dyn=0 rowshare=1 a_stages=3",
    "bf16_no_fat conv3_1":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv3_2":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv3_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=1 stages=4 epi_bufs=1 smem=218240 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv4_1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv4_2":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv4_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat loss1_conv1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv5_1":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv5_3":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat conv6_1":
        "kernel=conv_igemm_kernel<256, false> box=16x8x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat LFCN_1_5x5":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat LFCN_1_7x7":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat LFCN_2_5x5":
        "kernel=conv_igemm_kernel<64, false> box=32x4x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat LFCN_3_7x7":
        "kernel=conv_igemm_kernel<64, false> box=16x8x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat LFCN_4_5x5":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat LFCN_4_7x7":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat roi_c1":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_fat fc6":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_fat cls_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_fat bbox_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_fat roi_c1_nchw_f32":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_fat conv1_2_pool_full":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=1 smem=156864 dyn=0 rowshare=1 a_stages=4",
    "bf16_no_fat conv2_2_pool_full":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=1 fat=0 pool=1 stages=8 epi_bufs=2 smem=225472 dyn=0 rowshare=1 a_stages=3",
    "bf16_no_fat conv3_3_pool_full":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=1 stages=4 epi_bufs=1 smem=218240 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat n1_64":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=1 smem=152768 dyn=0 rowshare=1 a_stages=4",
    "bf16_no_fat n1_128_pool":
        "kernel=conv_igemm_kernel<128, false> box=32x4x1 terms=1 fat=0 pool=1 stages=5 epi_bufs=2 smem=205952 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat n1_odd_w_64":
        "kernel=conv_igemm_kernel<64, false> box=18x7x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat n1_odd_w_128":
        "kernel=conv_igemm_kernel<128, false> box=18x7x1 terms=1 fat=0 pool=0 stages=6 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat n1_odd_w_256":
        "kernel=conv_igemm_kernel<256, false> box=5x25x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat n3_odd_w_1x1":
        "kernel=conv_igemm_kernel<256, false> box=41x1x3 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat n2_odd_w_nchw":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat n1_head_3x1":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_fat narrow_cout_32":
        "kernel=conv_igemm_kernel<32, false> box=16x8x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=164992 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv1_2":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=1 stages=7 epi_bufs=2 smem=214144 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv2_1":
        "kernel=conv_igemm_kernel<128, false> box=128x1x1 terms=1 fat=0 pool=0 stages=6 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv2_2":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=1 fat=0 pool=1 stages=5 epi_bufs=2 smem=205952 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv3_1":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv3_2":
        "kernel=conv_igemm_kernel<256, false> box=128x1x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv3_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=1 stages=4 epi_bufs=1 smem=218240 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv4_1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv4_2":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv4_3":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare loss1_conv1":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv5_1":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv5_3":
        "kernel=conv_igemm_kernel<256, false> box=32x4x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv6_1":
        "kernel=conv_igemm_kernel<256, false> box=16x8x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare LFCN_1_5x5":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare LFCN_1_7x7":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare LFCN_2_5x5":
        "kernel=conv_igemm_kernel<64, false> box=32x4x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare LFCN_3_7x7":
        "kernel=conv_igemm_kernel<64, false> box=16x8x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare LFCN_4_5x5":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare LFCN_4_7x7":
        "kernel=conv_igemm_kernel<64, false> box=8x4x4 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare roi_c1":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_rowshare fc6":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_rowshare cls_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_rowshare bbox_pred":
        "kernel=conv_igemm_kernel<64, false> box=1x1x128 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_rowshare roi_c1_nchw_f32":
        "kernel=conv_igemm_kernel<256, false> box=1x1x128 terms=1 fat=0 pool=0 stages=4 epi_bufs=0 smem=197760 dyn=1 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv1_2_pool_full":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=1 stages=7 epi_bufs=2 smem=214144 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv2_2_pool_full":
        "kernel=conv_igemm_kernel<128, false> box=64x2x1 terms=1 fat=0 pool=1 stages=5 epi_bufs=2 smem=205952 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare conv3_3_pool_full":
        "kernel=conv_igemm_kernel<256, false> box=64x2x1 terms=1 fat=0 pool=1 stages=4 epi_bufs=1 smem=218240 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n1_64":
        "kernel=conv_igemm_kernel<64, false> box=64x2x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n1_128_pool":
        "kernel=conv_igemm_kernel<128, false> box=32x4x1 terms=1 fat=0 pool=1 stages=5 epi_bufs=2 smem=205952 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n1_odd_w_64":
        "kernel=conv_igemm_kernel<64, false> box=18x7x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n1_odd_w_128":
        "kernel=conv_igemm_kernel<128, false> box=18x7x1 terms=1 fat=0 pool=0 stages=6 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n1_odd_w_256":
        "kernel=conv_igemm_kernel<256, false> box=5x25x1 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n3_odd_w_1x1":
        "kernel=conv_igemm_kernel<256, false> box=41x1x3 terms=1 fat=0 pool=0 stages=4 epi_bufs=2 smem=230528 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n2_odd_w_nchw":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare n1_head_3x1":
        "kernel=conv_igemm_kernel<64, false> box=41x3x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=197760 dyn=0 rowshare=0 a_stages=0",
    "bf16_no_rowshare narrow_cout_32":
        "kernel=conv_igemm_kernel<32, false> box=16x8x1 terms=1 fat=0 pool=0 stages=8 epi_bufs=0 smem=164992 dyn=0 rowshare=0 a_stages=0",
}
