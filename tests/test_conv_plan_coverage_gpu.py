"""Every pinned launch plan of conv_igemm_kernel run and checked, at the sizes of tests/conv_plan_cases.py (whose CPU
test holds each entry to its pinned plan string).

Per entry, under its config's switches, the launch is the descriptor that was described, with outputs pre-filled with
a NaN sentinel no kernel produces:
- every element up to Cout_pad is written, and channels [Cout, Cout_pad) (zero weights, zero bias) are exactly +0 in
  hi and lo, since the next layer multiplies them by zero weights and a NaN there would poison it;
- the values match an fp64 convolution at test_conv_gpu.py's bars: split 1e-4 (|ref| + rms); plain bf16 against the
  rounded operands, 2^-8 relative + 1e-5 rms (widened as sqrt(K / 512) beyond K = 512 for the fp32 accumulation);
- pooled planes equal mscnn_pool_forward of the stored planes bit for bit, in the store-both and pool-only forms;
- the pixel-major head form (NHWC fp32) is also summed by mscnn_head_gather and compared with the k x k convolution;
- a dyn layer run with a count below N equals the run without a count below it, and keeps the sentinel from the count
  rounded up to the box's images;
- a second launch is bit-identical."""
import zlib
from dataclasses import replace

import pytest
import torch
import torch.nn.functional as F

import conv_plan_cases as cpc
from test_conv_gpu import _report

pytestmark = pytest.mark.gpu

SENT_BF16 = 0x7FBF          # a quiet NaN no kernel produces
SENT_F32 = 0x7FC00001
ENTRIES = cpc.entries()


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _sentinel_like(shape, dtype, device):
    t = torch.empty(shape, dtype=dtype, device=device)
    _bits(t).fill_(SENT_BF16 if dtype == torch.bfloat16 else SENT_F32)
    return t


def _unwritten(t):
    return int((_bits(t) == (SENT_BF16 if t.dtype == torch.bfloat16 else SENT_F32)).sum())


class Launch:
    """Operands of one entry and its launches through mscnn_conv_forward on exactly the descriptor cpc.desc builds."""

    def __init__(self, e, device):
        from mscnn_b200 import capi, ops
        self.e, L = e, e.layer
        self.ho, self.wo = cpc.out_hw(L, e.h, e.w)
        g = torch.Generator(device="cpu").manual_seed(zlib.crc32(e.id.encode()))
        cin_g = L.cin // L.group
        self.x = torch.randn((e.n, L.cin, e.h, e.w), generator=g).to(device)
        b = torch.randn((L.cout,), generator=g) * 0.1
        if L.out == cpc.NHWC_F32:
            # the k x k proposal head as a k x 1 convolution with k * cout columns (mscnn_pack_head_weights)
            k = L.kh
            self.head_cout = 9 if k * 9 <= L.cout_pad else L.cout_pad // k
            self.wt = (torch.randn((self.head_cout, L.cin, k, k), generator=g) * 0.02).to(device)
            self.b = b[: self.head_cout].to(device)
            hi = torch.empty((L.cout_pad, k, 1, L.cin), dtype=torch.bfloat16, device=device)
            lo = torch.empty_like(hi) if e.split else None
            capi.check(capi.lib().mscnn_pack_head_weights(capi.ptr(self.wt), capi.ptr(hi), capi.ptr(lo), self.head_cout,
                                                          L.cin, k, L.cout_pad, L.cin, ops._stream()), "pack_head_weights")
            self.wp = ops.PackedWeights(hi, lo, torch.zeros(L.cout_pad, dtype=torch.float32, device=device), L.cout, k, 1)
            # the same k x 1 convolution as [dx * cout + co][c][dy][0], zero rows to Cout_pad
            w2 = torch.zeros((L.cout_pad, L.cin, k, 1), device=device)
            w2[: k * self.head_cout] = self.wt.permute(3, 0, 1, 2).reshape(k * self.head_cout, L.cin, k, 1)
            self.wref, self.bref = w2, torch.zeros(L.cout_pad, device=device)
        else:
            self.wt = (torch.randn((L.cout, cin_g, L.kh, L.kw), generator=g) * (2.0 / (cin_g * L.kh * L.kw)) ** 0.5).to(device)
            self.b = b.to(device)
            self.wp = ops.pack_conv_weights(self.wt, self.b, e.split, cout_pad=L.cout_pad, cin_pad=cin_g)
            self.wref, self.bref = self.wt, self.b
        self.xp = ops.nchw_to_planes(self.x, e.split)
        assert self.xp.hi.shape[3] == L.cin and tuple(self.wp.hi.shape[1:]) == (L.kh, L.kw, cin_g)

    def outputs(self, pool_only=None):
        e, L, dev = self.e, self.e.layer, self.x.device
        out = {}
        if L.out == cpc.BF16:
            store = L.store_full if pool_only is None else not pool_only
            planes = ["hi", "lo"] if e.split else ["hi"]
            if store or not L.pool:
                for p in planes:
                    out["y_" + p] = _sentinel_like((e.n, self.ho, self.wo, L.cout_pad), torch.bfloat16, dev)
            if L.pool:
                for p in planes:
                    out["pool_" + p] = _sentinel_like((e.n, self.ho // 2, self.wo // 2, L.cout_pad), torch.bfloat16, dev)
        elif L.out == cpc.NCHW_F32:
            out["y_f32"] = _sentinel_like((e.n, L.cout, self.ho, self.wo), torch.float32, dev)
        else:
            out["y_f32"] = _sentinel_like((e.n, self.ho, self.wo, L.cout_pad), torch.float32, dev)
        return out

    def run(self, pool_only=None, count=None):
        """count: the device row count of a dyn layer (None: the launch without one, dyn=0)."""
        from mscnn_b200 import capi, ops
        e = self.e
        layer = e.layer if count is not None else replace(e.layer, dyn=False)
        out = self.outputs(pool_only)
        dyn = torch.tensor([count if count is not None else 0], dtype=torch.int32, device=self.x.device)
        ptrs = {"x_hi": capi.ptr(self.xp.hi), "x_lo": capi.ptr(self.xp.lo), "w_hi": capi.ptr(self.wp.hi),
                "w_lo": capi.ptr(self.wp.lo), "bias": capi.ptr(self.wp.bias), "dyn_n": capi.ptr(dyn)}
        ptrs.update({k: capi.ptr(v) for k, v in out.items()})
        d = cpc.desc(layer, e.split, e.n, e.h, e.w, ptrs=ptrs, pool_only=pool_only)
        rc, text = cpc.describe(d)
        want = cpc.pinned(e.key)
        assert rc == 0 and text == (want if layer.dyn else want.replace("dyn=1", "dyn=0")), (e.id, text)
        capi.check(capi.lib().mscnn_conv_forward(d, ops._stream()), "conv_forward")
        torch.cuda.synchronize()
        return out

    def ref(self):
        e, L = self.e, self.e.layer
        x, w = self.x.double(), self.wref.double()
        if not e.split:
            x, w = self.x.bfloat16().double(), self.wref.bfloat16().double()
        y = F.conv2d(x, w, self.bref.double(), stride=L.stride, padding=(L.pad_h, L.pad_w), dilation=L.dil,
                     groups=L.group)
        return torch.relu(y) if L.out == cpc.BF16 else y


def _check_values(e, name, got, ref):
    rms = float(ref.pow(2).mean().sqrt())
    if e.split:
        _report(f"{e.id} {name}", got, ref, 1e-4, 1e-4 * rms)
    else:
        # the fp32 accumulation over K adds error growing as sqrt(K): 1e-5 rms up to K = 512, 3e-5 at roi_c1's 4608
        # (the bar test_device_rows_gpu.py measured), 5e-5 at fc6's 12800
        L = e.layer
        k = L.cin // L.group * L.kh * L.kw
        _report(f"{e.id} {name}", got, ref, 2.0 ** -8, 1e-5 * max(1.0, (k / 512) ** 0.5) * rms)


def _planes_nchw(hi, lo, cout):
    v = hi.float() + (lo.float() if lo is not None else 0)
    return v[..., :cout].permute(0, 3, 1, 2)


def _check_written(e, out):
    L = e.layer
    for k, t in out.items():
        n = _unwritten(t)
        assert n == 0, f"{e.id}: {n}/{t.numel()} elements of {k} were not written"
        if k != "y_f32" and L.cout < L.cout_pad:
            pad = _bits(t[..., L.cout:])
            assert bool((pad == 0).all()), f"{e.id}: channels [{L.cout}, {L.cout_pad}) of {k} are not +0"


def _same(e, what, a, b):
    for k in a:
        if not torch.equal(_bits(a[k]), _bits(b[k])):
            d = (_bits(a[k]) != _bits(b[k])).nonzero()
            pytest.fail(f"{e.id}: {what}: {k} differs in {d.shape[0]} elements, first at {d[:4].tolist()}")


@pytest.mark.parametrize("e", ENTRIES, ids=[e.id.replace(" ", "-") for e in ENTRIES])
def test_pinned_plan_values(cuda, e, monkeypatch):
    from mscnn_b200 import capi, ops
    for k in ("MSCNN_NO_FAT", "MSCNN_NO_ROWSHARE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in e.env.items():
        monkeypatch.setenv(k, v)
    ops.reload_config()
    try:
        run = Launch(e, cuda)
        L = e.layer
        count = e.n if L.dyn else None
        out = run.run(count=count)
        _check_written(e, out)
        _same(e, "a second launch", out, run.run(count=count))
        ref = run.ref()

        if L.out == cpc.BF16:
            if L.pool:
                both = run.run(pool_only=False, count=count)
                only = run.run(pool_only=True, count=count)
                _check_written(e, both)
                _check_written(e, only)
                y = ops.Planes(both["y_hi"], both.get("y_lo"), L.cout)
                pooled = ops.pool_forward(y, 2, 2)
                torch.cuda.synchronize()
                for form in (both, only):
                    _same(e, "pooled planes vs mscnn_pool_forward of the stored planes", {"pool_hi": pooled.hi, **(
                        {"pool_lo": pooled.lo} if e.split else {})}, {k: form[k] for k in form if k.startswith("pool")})
                got = _planes_nchw(both["y_hi"], both.get("y_lo"), L.cout)
            else:
                got = _planes_nchw(out["y_hi"], out.get("y_lo"), L.cout)
            _check_values(e, "planes", got, ref)
        elif L.out == cpc.NCHW_F32:
            _check_values(e, "nchw_f32", out["y_f32"], ref)
        else:
            p = out["y_f32"]
            _check_values(e, "pixel-major rows", p.permute(0, 3, 1, 2), ref)
            k = L.kh
            assert bool((_bits(p[..., k * run.head_cout:]) == 0).all()), f"{e.id}: columns without a tap are not +0"
            y = torch.empty((e.n, run.head_cout, e.h, e.w), dtype=torch.float32, device=cuda)
            capi.check(capi.lib().mscnn_head_gather(capi.ptr(p), L.cout_pad, capi.ptr(run.b), capi.ptr(y), e.n, e.h,
                                                    e.w, run.head_cout, k, k // 2, ops._stream()), "head_gather")
            torch.cuda.synchronize()
            x, wt = (run.x, run.wt) if e.split else (run.x.bfloat16().float(), run.wt.bfloat16().float())
            _check_values(e, "gathered head", y, F.conv2d(x.double(), wt.double(), run.b.double(), padding=k // 2))

        if L.dyn:
            full = run.run(count=None)
            _same(e, "the launch without a count", out, full)
            bn = cpc.box(cpc.pinned(e.key))[2]
            c = e.n - bn - 3 if e.n > bn + 3 else e.n - 1
            part = run.run(count=c)
            trimmed = -(-c // bn) * bn
            for k in part:
                got, want = _bits(part[k]), _bits(full[k])
                assert torch.equal(got[:c], want[:c]), f"{e.id} count={c}: rows below the count differ in {k}"
                tail = got[trimmed:]
                assert _unwritten(part[k][trimmed:]) == tail.numel(), f"{e.id} count={c}: rows from {trimmed} of {k} were written"
                mid = (got[c:trimmed] == want[c:trimmed]) | (got[c:trimmed] == (SENT_BF16 if part[k].dtype == torch.bfloat16 else SENT_F32))
                assert bool(mid.all()), (e.id, c, k)
    finally:
        monkeypatch.undo()
        ops.reload_config()
