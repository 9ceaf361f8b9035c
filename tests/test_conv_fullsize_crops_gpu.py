"""Every convolution of test_conv_layout_cpu.CASES at its full size, held bit for bit to launches of the same layer on
crops of its input.

Each output pixel's sum order depends on the layer alone: (term, dy, channel chunk, dx), then the MMA order inside a K
step, fixed by BLOCK_N, FAT and the number of terms (DESIGN.md section 4.1), not by the pixel box, ring depth, row-share,
tile position or batch composition.  So a full-size launch, whose persistent CTAs walk hundreds of tiles with rings
that wrap thousands of times, must equal the same layer launched on a crop of its input: the crop's input window with
its halo, zero-filled outside the image (TMA's zero fill is the padding, so the products are the same), at pad 0.  The
crops tile the whole output, with edges off the full launch's box grid (pooled crops start at even coordinates), and
one crop in 16 is also compared with fp64 so the chain stays anchored.  The row-count layers (ROI head and
InnerProducts, R = 16000) are held to row subsets of 1, 127, 128 and 129 rows and to a permutation of all rows instead,
and run once more with a device count of 12345.

Inputs are seeded random bf16 planes (hi and lo on the fp32-faithful path), default switches.  conv1_2 split holds
about 8 GB of input and output planes."""
from dataclasses import replace

import pytest
import torch
import torch.nn.functional as F

import conv_plan_cases as cpc
from test_conv_gpu import _report
from test_conv_layout_cpu import CASES

pytestmark = pytest.mark.gpu

SENT_BF16 = 0x7FBF
SENT_F32 = 0x7FC00001
CROP_H, CROP_W, CROP_N = 61, 251, 5      # off every box grid: 61 and 251 are odd primes, 5 divides no box_n
ROW_CASES = [c for c in CASES if CASES[c][13]]
CROP_CASES = [c for c in CASES if not CASES[c][13]]
DYN_COUNT = 12345


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _sent(dtype):
    return SENT_BF16 if dtype == torch.bfloat16 else SENT_F32


class Layer:
    """Seeded bf16 operand planes of one case and launches of it on any input window."""

    def __init__(self, case, split, device):
        self.case, self.split, self.dev = case, split, device
        self.L = cpc.layer_of(case)
        L = self.L
        n, _, h, w = CASES[case][:4]
        self.n, self.h, self.w = n, h, w
        g = torch.Generator(device=device).manual_seed(sum(map(ord, case)) + (7 if split else 0))
        self.x_hi = torch.randn((n, h, w, L.cin), generator=g, device=device).bfloat16()
        self.x_lo = (torch.randn((n, h, w, L.cin), generator=g, device=device) * 2.0 ** -9).bfloat16() if split else None
        k = L.cin * L.kh * L.kw
        scale = (2.0 / k) ** 0.5
        self.w_hi = (torch.randn((L.cout_pad, L.kh, L.kw, L.cin), generator=g, device=device) * scale).bfloat16()
        self.w_lo = (torch.randn((L.cout_pad, L.kh, L.kw, L.cin), generator=g, device=device) * scale * 2.0 ** -9).bfloat16() if split else None
        self.bias = torch.randn((L.cout_pad,), generator=g, device=device) * 0.1
        self.w_hi[L.cout:] = 0
        if split:
            self.w_lo[L.cout:] = 0
        self.bias[L.cout:] = 0

    def launch(self, layer, x_hi, x_lo, count=None):
        """Outputs (sentinel-filled first) of `layer` on the planes x_hi / x_lo: a dict like the descriptor's fields."""
        from mscnn_b200 import capi, ops
        L, split = layer, self.split
        n, h, w = x_hi.shape[:3]
        ho, wo = cpc.out_hw(L, h, w)
        out = {}
        planes = ["hi", "lo"] if split else ["hi"]
        if L.out == cpc.BF16:
            if L.store_full or not L.pool:
                for p in planes:
                    out["y_" + p] = torch.empty((n, ho, wo, L.cout_pad), dtype=torch.bfloat16, device=self.dev)
            if L.pool:
                for p in planes:
                    out["pool_" + p] = torch.empty((n, ho // 2, wo // 2, L.cout_pad), dtype=torch.bfloat16, device=self.dev)
        elif L.out == cpc.NCHW_F32:
            out["y_f32"] = torch.empty((n, L.cout, ho, wo), dtype=torch.float32, device=self.dev)
        else:
            out["y_f32"] = torch.empty((n, ho, wo, L.cout_pad), dtype=torch.float32, device=self.dev)
        for t in out.values():
            _bits(t).fill_(_sent(t.dtype))
        dyn = torch.tensor([n if count is None else count], dtype=torch.int32, device=self.dev)
        ptrs = {"x_hi": capi.ptr(x_hi), "x_lo": capi.ptr(x_lo), "w_hi": capi.ptr(self.w_hi), "w_lo": capi.ptr(self.w_lo),
                "bias": capi.ptr(self.bias), "dyn_n": capi.ptr(dyn), **{k: capi.ptr(v) for k, v in out.items()}}
        d = cpc.desc(L, split, n, h, w, ptrs=ptrs)
        capi.check(capi.lib().mscnn_conv_forward(d, ops._stream()), "conv_forward")
        torch.cuda.synchronize()
        return out

    def fp64(self, x_hi, x_lo, layer):
        """fp64 convolution (+ReLU for planes, + 2x2 max pooling for pooled planes) of the operand values."""
        x = x_hi.double() + (x_lo.double() if x_lo is not None else 0)
        wt = self.w_hi.double() + (self.w_lo.double() if self.w_lo is not None else 0)
        L = layer
        y = F.conv2d(x.permute(0, 3, 1, 2), wt[: L.cout].permute(0, 3, 1, 2), self.bias[: L.cout].double(),
                     padding=(L.pad_h, L.pad_w))
        return torch.relu(y) if L.out == cpc.BF16 else y

    def check_fp64(self, what, out, x_hi, x_lo, layer):
        L = layer
        ref = self.fp64(x_hi, x_lo, layer)
        k = L.cin * L.kh * L.kw
        for name, t in out.items():
            if name.endswith("_lo"):
                continue
            if name == "y_f32":
                got = t if L.out == cpc.NCHW_F32 else t.permute(0, 3, 1, 2)[:, : L.cout]
                r = ref
            else:
                lo = out.get(name.replace("_hi", "_lo"))
                got = (t.float() + (lo.float() if lo is not None else 0))[..., : L.cout].permute(0, 3, 1, 2)
                r = F.max_pool2d(ref, 2) if name.startswith("pool") else ref
            rms = float(r.pow(2).mean().sqrt())
            if self.split:
                _report(f"{what} {name}", got, r, 1e-4, 1e-4 * rms)
            else:
                _report(f"{what} {name}", got, r, 2.0 ** -8, 1e-5 * max(1.0, (k / 512) ** 0.5) * rms)


def _crop_input(x, n0, n1, y0, y1, x0, x1, L):
    """The input window of output rows [y0, y1) and columns [x0, x1), halo included, zero outside the image."""
    if x is None:
        return None
    _, h, w, c = x.shape
    iy0, iy1, ix0, ix1 = y0 - L.pad_h, y1 - 1 - L.pad_h + L.kh, x0 - L.pad_w, x1 - 1 - L.pad_w + L.kw
    out = torch.zeros((n1 - n0, iy1 - iy0, ix1 - ix0, c), dtype=x.dtype, device=x.device)
    sy0, sy1, sx0, sx1 = max(iy0, 0), min(iy1, h), max(ix0, 0), min(ix1, w)
    out[:, sy0 - iy0: sy1 - iy0, sx0 - ix0: sx1 - ix0] = x[n0:n1, sy0:sy1, sx0:sx1]
    return out


def _full_window(name, t, n0, n1, y0, y1, x0, x1, L):
    if name.startswith("pool"):
        return t[n0:n1, y0 // 2: y1 // 2, x0 // 2: x1 // 2]
    if name == "y_f32" and L.out == cpc.NCHW_F32:
        return t[n0:n1, :, y0:y1, x0:x1]
    return t[n0:n1, y0:y1, x0:x1]


def _equal(what, a, b):
    if not torch.equal(_bits(a), _bits(b)):
        d = (_bits(a) != _bits(b)).nonzero()
        pytest.fail(f"{what}: {d.shape[0]}/{a.numel()} elements differ from the full launch, first at {d[:4].tolist()}")


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", CROP_CASES)
def test_full_size_equals_its_crops(cuda, case, split):
    lay = Layer(case, split, cuda)
    L = lay.L
    full = lay.launch(L, lay.x_hi, lay.x_lo)
    for name, t in full.items():
        assert not bool((_bits(t) == _sent(t.dtype)).any()), f"{case}: {name} not entirely written"
    ho, wo = cpc.out_hw(L, lay.h, lay.w)
    ch, cw = (CROP_H + 1, CROP_W - 1) if L.pool else (CROP_H, CROP_W)
    crop_layer = replace(L, pad_h=0, pad_w=0)
    i = 0
    for n0 in range(0, lay.n, CROP_N):
        n1 = min(n0 + CROP_N, lay.n)
        for y0 in range(0, ho, ch):
            y1 = min(y0 + ch, ho)
            for x0 in range(0, wo, cw):
                x1 = min(x0 + cw, wo)
                xh = _crop_input(lay.x_hi, n0, n1, y0, y1, x0, x1, L)
                xl = _crop_input(lay.x_lo, n0, n1, y0, y1, x0, x1, L)
                got = lay.launch(crop_layer, xh, xl)
                what = f"{case} crop n[{n0}:{n1}] y[{y0}:{y1}] x[{x0}:{x1}]"
                for name, t in got.items():
                    _equal(f"{what} {name}", t, _full_window(name, full[name], n0, n1, y0, y1, x0, x1, L))
                if i % 16 == 0:
                    # one image of the crop: the fp64 reference of the whole crop would dominate the test's time
                    lay.check_fp64(what, {k: v[:1] for k, v in got.items()}, xh[:1], None if xl is None else xl[:1],
                                   crop_layer)
                i += 1


@pytest.mark.parametrize("split", [True, False], ids=["split", "bf16"])
@pytest.mark.parametrize("case", ROW_CASES)
def test_row_layers_equal_their_row_subsets(cuda, case, split):
    lay = Layer(case, split, cuda)
    L = lay.L
    full = lay.launch(L, lay.x_hi, lay.x_lo)
    for name, t in full.items():
        assert not bool((_bits(t) == _sent(t.dtype)).any()), f"{case}: {name} not entirely written"
    g = torch.Generator(device="cpu").manual_seed(77)
    perm = torch.randperm(lay.n, generator=g).to(cuda)
    subsets = {"first row": perm.new_tensor([0]), "127 rows": perm[:127], "128 rows": perm[127:255],
               "129 rows": perm[255:384], "all rows permuted": perm}
    for what, idx in subsets.items():
        xh = lay.x_hi[idx].contiguous()
        xl = None if lay.x_lo is None else lay.x_lo[idx].contiguous()
        got = lay.launch(L, xh, xl)
        for name, t in got.items():
            _equal(f"{case} {what} {name}", t, full[name][idx])
        if what in ("127 rows", "129 rows"):
            lay.check_fp64(f"{case} {what}", got, xh, xl, L)
    part = lay.launch(L, lay.x_hi, lay.x_lo, count=DYN_COUNT)
    bn = cpc.box(cpc.describe(cpc.desc(L, split, lay.n, lay.h, lay.w))[1])[2]
    trimmed = -(-DYN_COUNT // bn) * bn
    for name, t in part.items():
        _equal(f"{case} count={DYN_COUNT} rows below the count, {name}", t[:DYN_COUNT], full[name][:DYN_COUNT])
        assert bool((_bits(t[trimmed:]) == _sent(t.dtype)).all()), f"{case}: rows from {trimmed} of {name} were written"
        mid, want = _bits(t[DYN_COUNT:trimmed]), _bits(full[name][DYN_COUNT:trimmed])
        assert bool(((mid == want) | (mid == _sent(t.dtype))).all())
