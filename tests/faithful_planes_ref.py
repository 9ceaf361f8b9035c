"""Shared by tests/test_faithful_planes_cpu.py and tests/test_faithful_planes_gpu.py: inputs whose split into bf16 planes
has a live lo plane, the rounding store8 applies to a kernel's fp32 result, the ROI set of the plane-kernel tests, the
bin windows ROIPooling walks, and global AVE pooling restated in the order global_pool_kernel sums.

A split activation is x = hi + lo with hi = bf16_rn(x) and lo = bf16_rn(x - hi) (mscnn_nchw_f32_to_planes); the kernels
between two convolutions add hi + lo in fp32, which is exact.  torch's CPU float -> bfloat16 conversion rounds to nearest
even, as __float2bfloat16_rn does."""
import numpy as np
import torch

F32 = np.float32
TIE_STEP = 2.0 ** -12        # lo steps of the planted ties: 1 + k 2^-12 keeps hi = 1 for -7 <= k <= 15
TIE_K = np.arange(-7, 16)
TIE_PATCH = 4                # planted tie patches are 4 x 4 pixels, in every channel


def bf16_rn(x) -> np.ndarray:
    """fp32 -> the fp32 value of its bf16 round-to-nearest-even."""
    return torch.from_numpy(np.ascontiguousarray(x, dtype=F32)).bfloat16().float().numpy()


def split_planes(x):
    """(hi, lo) of fp32 x as fp32 arrays: the planes mscnn_nchw_f32_to_planes writes."""
    x = np.asarray(x, dtype=F32)
    hi = bf16_rn(x)
    return hi, bf16_rn(x - hi)


def stored(r, split: bool) -> np.ndarray:
    """What store8 keeps of a kernel's fp32 result r, read back as planes_to_nchw does: hi' + lo' with hi' = bf16_rn(r),
    lo' = bf16_rn(r - hi') (split), or hi' alone."""
    hi, lo = split_planes(r)
    return (hi + lo).astype(F32) if split else hi


def half_ulp(hi) -> np.ndarray:
    """Half a bf16 ulp of the (non-zero, normal) bf16 values hi, as fp32."""
    e = np.floor(np.log2(np.abs(np.asarray(hi, dtype=np.float64))))
    return (2.0 ** (e - 8)).astype(F32)


def faithful_input(rng, shape, kind: str, ties: int = 6, halfway: float = 0.03, neg_zero: int = 8) -> np.ndarray:
    """fp32 NCHW whose split keeps a non-zero lo on >= 90 % of the elements.

    kind "signed": standard normal.  kind "relu": max(z + 1.4, 0), non-negative with ~8 % zeros, like a post-ReLU map.
    Planted on top, per image:
      * `ties` patches of 4 x 4 pixels in every channel holding s (1 + k 2^-12), k a per-channel permutation of -7..15
        and s a power of two above the map's values: within any window over such a patch the largest values share hi
        and differ in lo only, with lo of either sign;
      * a fraction `halfway` of the elements moved to m + 1/2 ulp(m) for their own bf16 value m: the split rounds them
        to even, so lo is exactly +-1/2 ulp of hi;
      * (signed only) `neg_zero` elements set to -0.0."""
    n, c, h, w = shape
    if kind == "signed":
        x = rng.standard_normal(shape).astype(F32)
    elif kind == "relu":
        x = np.maximum(rng.standard_normal(shape) + 1.4, 0.0).astype(F32)
    else:
        raise ValueError(kind)
    flat = x.reshape(-1)
    pick = rng.choice(flat.size, int(halfway * flat.size), replace=False)
    m = bf16_rn(flat[pick])
    m[m == 0] = F32(1.0)
    flat[pick] = m + np.sign(m) * half_ulp(m)
    p = TIE_PATCH
    for i in range(n):
        for _ in range(ties if h >= p and w >= p else 0):
            y0, x0 = rng.integers(0, h - p + 1), rng.integers(0, w - p + 1)
            scale = F32(2.0 ** rng.integers(3, 5))
            ks = np.stack([rng.permutation(TIE_K)[: p * p] for _ in range(c)]).reshape(c, p, p)
            x[i, :, y0:y0 + p, x0:x0 + p] = (scale * (1.0 + ks * TIE_STEP)).astype(F32)
    if kind == "signed" and neg_zero:
        flat[rng.choice(flat.size, neg_zero, replace=False)] = F32(-0.0)
    return x


def special_rois(rng, n, img_w, img_h, r):
    """Random boxes plus the edge ROIs of the layer tests: the dummy ROI, a malformed one (x2 < x1), one outside the
    image (empty bins), one on half-pixel coordinates (round() away from zero), the full-map box, and a tenth of
    boxes smaller than a feature-map pixel."""
    x1 = rng.uniform(-20, img_w, r); y1 = rng.uniform(-20, img_h, r)
    bw = rng.uniform(1, 300, r); bh = rng.uniform(1, 200, r)
    rois = np.stack([rng.integers(0, n, r), x1, y1, x1 + bw, y1 + bh], axis=1).astype(F32)
    k = r // 10
    rois[5:5 + k, 3] = rois[5:5 + k, 1] + rng.uniform(0, 6, k)
    rois[5:5 + k, 4] = rois[5:5 + k, 2] + rng.uniform(0, 6, k)
    rois[0] = [0, 1, 1, 10, 10]
    rois[1] = [1 % n, 50, 40, 30, 20]
    rois[2] = [0, img_w + 100, img_h + 100, img_w + 200, img_h + 200]
    rois[3] = [1 % n, 3.5, 4.5, 4.5, 5.5]
    rois[4] = [0, 0, 0, img_w - 1, img_h - 1]
    return rois


def roi_pool_windows(rois, h, w, pooled_h, pooled_w, scale, pad_ratio) -> np.ndarray:
    """Pixel count of every ROIPooling bin window [R, pooled_h, pooled_w] (0: an empty bin), with the fp32 geometry of
    roi_pooling_layer.cpp:66-110 (and of roi_pool_kernel)."""
    q = np.asarray(rois, dtype=F32).reshape(-1, 5)
    one, s, pr = F32(1), F32(scale), F32(pad_ratio)
    pad_w = (q[:, 3] - q[:, 1] + one) * pr
    pad_h = (q[:, 4] - q[:, 2] + one) * pr

    def rnd(v):                                           # roundf: half away from zero
        return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)
    sw, sh = rnd((q[:, 1] - pad_w) * s), rnd((q[:, 2] - pad_h) * s)
    ew, eh = rnd((q[:, 3] + pad_w) * s), rnd((q[:, 4] + pad_h) * s)
    roi_h, roi_w = np.maximum(eh - sh + 1, 1), np.maximum(ew - sw + 1, 1)
    bin_h, bin_w = roi_h.astype(F32) / F32(pooled_h), roi_w.astype(F32) / F32(pooled_w)
    ph = np.arange(pooled_h, dtype=F32)[None, :]
    pw = np.arange(pooled_w, dtype=F32)[None, :]
    hs = np.clip(np.floor(ph * bin_h[:, None]).astype(np.int64) + sh[:, None], 0, h)
    he = np.clip(np.ceil((ph + 1) * bin_h[:, None]).astype(np.int64) + sh[:, None], 0, h)
    ws = np.clip(np.floor(pw * bin_w[:, None]).astype(np.int64) + sw[:, None], 0, w)
    we = np.clip(np.ceil((pw + 1) * bin_w[:, None]).astype(np.int64) + sw[:, None], 0, w)
    return np.maximum(he - hs, 0)[:, :, None] * np.maximum(we - ws, 0)[:, None, :]


GLOBAL_SLICES = 32


def global_ave_kernel_order(x) -> np.ndarray:
    """Global AVE pooling of fp32 x [N, C, H, W] summed as global_pool_kernel sums (H W >= 32): slice s adds pixels s,
    s + 32, s + 64, ... in turn, slice 0 then adds the slices' sums 1..31 to its own, and the total is divided by H W.
    Every step an fp32 add -> [N, C, 1, 1]."""
    x = np.asarray(x, dtype=F32)
    n, c, h, w = x.shape
    hw = h * w
    assert hw >= GLOBAL_SLICES
    flat = x.reshape(n, c, hw)
    parts = []
    for s in range(GLOBAL_SLICES):
        acc = np.zeros((n, c), dtype=F32)
        for px in range(s, hw, GLOBAL_SLICES):
            acc = acc + flat[:, :, px]
        parts.append(acc)
    acc = parts[0]
    for p in parts[1:]:
        acc = acc + p
    return (acc / F32(hw)).reshape(n, c, 1, 1)
