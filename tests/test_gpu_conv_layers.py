"""GPU: each conv layer of tests/test_conv_layer_host.py run through the executors' own expansions (dmd_conv_layer_fprop /
_dgrad / _wgrad: K-split chunks, split-fp16 passes, backward-data chunks, weight-gradient blocks; packs from
dmd_conv_layer_pack) against float64 references of the same op, with the bounds the single-launch tests measured:

- fp16-operand launches (fp16 forward, dgrad, wgrad): 2e-5 relative RMS against float64 on fp16-rounded operands and 2e-3
  against the exact fp32 operands (tests/test_gpu_conv.py, tests/test_gpu_wgrad.py);
- split-fp16 forwards (one-launch chunks, three passes, chunked three passes): 5e-6 against float64 on the exact operands
  (test_conv_precise_split_fp16), while the same layer with fp16 operands is off by more than 2e-5 there, so a chunk or pass
  that falls back to fp16 accuracy fails.

Every call starts from NaN-filled or pre-filled outputs, so the first launch must assign and every later one accumulate; the
forward's statistics must be the sums of the output it produced (all chunks in); dgrad writes only its source's channels; the
weight gradient leaves the columns of the other concat source bitwise alone; and two runs give the same bytes."""
import math

import pytest
import torch
import torch.nn.functional as F

from diamond_b200 import _lib
from test_conv_layer_host import LAYERS, sources

pytestmark = pytest.mark.gpu

F64 = torch.float64
FP16_TOL, FP32_TOL = 2e-5, 2e-3     # tests/test_gpu_conv.py test_conv_plain, tests/test_gpu_wgrad.py
SPLIT_TOL = 5e-6                    # tests/test_gpu_conv.py test_conv_precise_split_fp16
STATS_PREFILL = 0.25

# (B, H, W): 8 x 8 at B = 5 puts several images in one 128-position tile; 24 x 40 is not square.  The stride-2 Downsample
# runs at 16 x 16 in place of 8 x 8
SIZES = [(5, 8, 8), (2, 24, 40)]
DOWN_SIZES = [(5, 16, 16), (2, 24, 40)]
FWD_LAYERS = [n for n in LAYERS if n != "conv_out"]
DGRAD_LAYERS = [n for n in LAYERS if LAYERS[n]["dgrad"] and n != "conv_out"]


def _cases(names):
    return [(n, s) for n in names for s in (DOWN_SIZES if LAYERS[n].get("stride", 1) == 2 else SIZES)]


def _id(c):
    return f"{c[0]}-{'x'.join(map(str, c[1]))}"


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-300))


def _h(t):
    return t.half().to(t.dtype)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


class _Case:
    """A layer at one size: its inputs (NHWC, stored channels; the padding channels of a source hold stale values, which the
    packs' zero rows and the blocks' channel counts must keep out), the torch weight and bias, and its packs."""

    def __init__(self, name, b, h, w, seed, dev):
        from diamond_b200 import ops

        self.name, self.b, self.h, self.w = name, b, h, w
        e = LAYERS[name]
        self.cout, self.cin_real, taps, self.c0_real, self.c0_store, self.c1, self.split, _ = e["args"]
        self.stride, self.k = e.get("stride", 1), 3 if taps == 9 else 1
        self.ho, self.wo = h // self.stride, w // self.stride
        self.layer = ops.ConvLayer(*e["args"])
        self.srcs = sources(name)
        g = torch.Generator(device=dev).manual_seed(seed)
        self.x = torch.randn(b, h, w, self.c0_store + self.c1, device=dev, generator=g)
        self.x_real = torch.cat([self.x[..., :self.c0_real], self.x[..., self.c0_store:]], -1)
        self.wt = torch.randn(self.cout, self.cin_real, self.k, self.k, device=dev, generator=g) / math.sqrt(self.cin_real * taps)
        self.bias = 0.1 * torch.randn(self.cout, device=dev, generator=g)
        self.gy = torch.randn(b, self.ho, self.wo, ops.round_up(self.cout, 8), device=dev, generator=g)   # padding: stale
        self.gen = g
        self.packed = self.layer.pack(self.wt)

    def source(self, k):
        stored, _, _ = self.srcs[k]
        lo = sum(s for s, _, _ in self.srcs[:k])
        return self.x[..., lo:lo + stored].contiguous()

    def conv_ref(self, fp16):
        x, w = (_h(self.x_real), _h(self.wt)) if fp16 else (self.x_real, self.wt)
        y = F.conv2d(_nchw(x).to(F64), w.to(F64), self.bias.to(F64), stride=self.stride, padding=self.k // 2)
        return _nhwc(y)

    def gy_real(self, fp16):
        g = self.gy[..., :self.cout]
        return _nchw(_h(g) if fp16 else g).to(F64)

    def dgrad_ref(self, fp16):
        w = (_h(self.wt) if fp16 else self.wt).to(F64)
        gx = torch.nn.grad.conv2d_input((self.b, self.cin_real, self.h, self.w), w, self.gy_real(fp16), stride=self.stride,
                                        padding=self.k // 2)
        return _nhwc(gx)

    def wgrad_ref(self, fp16):
        x = _nchw(_h(self.x_real) if fp16 else self.x_real).to(F64)
        gw = torch.nn.grad.conv2d_weight(x, tuple(self.wt.shape), self.gy_real(fp16), stride=self.stride, padding=self.k // 2)
        return gw.reshape(self.cout, self.cin_real, -1)

    def gy_operand(self, scale=1.0):
        """The PLC16 gradient operand at the conv input size (a stride-2 conv's gradient zero-inserted)."""
        from diamond_b200 import ops

        return ops.prep_act((self.gy[..., :] * scale).contiguous(), upsample=2 if self.stride == 2 else False)[0]


def _operands(c):
    from diamond_b200 import ops

    s0, s1 = c.source(0), (c.source(1) if c.c1 else None)
    res = ops.prep_act(s0, src1=s1, split=c.split)
    lo0, lo1 = (res[6], res[7]) if c.split else (None, None)
    return res[0], res[1], lo0, lo1


@pytest.mark.parametrize("case", _cases(FWD_LAYERS), ids=_id)
def test_forward_against_float64(case):
    dev = _dev()
    name, (b, h, w) = case
    c = _Case(name, b, h, w, 101 + b + h + w, dev)
    n0, n1, lo0, lo1 = _operands(c)
    ref, ref16 = c.conv_ref(False), c.conv_ref(True)
    fp16_err = _rel(ref16, ref)
    gs = 32 if c.cout % 32 == 0 else 0
    for residual in (None, torch.randn(b, c.ho, c.wo, c.cout, device=dev, generator=c.gen)):
        outs = []
        for run in range(2):
            out = torch.full((b, c.ho, c.wo, c.cout), float("nan"), device=dev)
            st = torch.full((b, c.cout // gs, 2), STATS_PREFILL, device=dev, dtype=F64) if gs else None
            c.layer.fprop(c.packed, n0, n1, b, h, w, out, lo0=lo0, lo1=lo1, stride=c.stride, bias=c.bias, residual=residual,
                          ostats=st, out_gs=gs)
            outs.append((out, st))
        torch.cuda.synchronize()
        (out, st), (out2, _) = outs
        want, want16 = (ref, ref16) if residual is None else (ref + residual.to(F64), ref16 + residual.to(F64))
        assert torch.isfinite(out).all(), "a launch left NaN behind: the first one must assign every output"
        e32, e16 = _rel(out, want), _rel(out, want16)
        print(f"{name} B={b} {h}x{w} residual={residual is not None}: rel RMS vs exact {e32:.2e}, vs fp16 operands {e16:.2e} "
              f"(fp16-operand error of the layer {fp16_err:.2e})")
        if c.split:
            assert e32 < SPLIT_TOL, (e32, fp16_err)
            assert fp16_err > FP16_TOL, fp16_err   # the bound tells the split-fp16 path from an fp16-operand one
        else:
            assert e16 < FP16_TOL, e16
            assert e32 < FP32_TOL, e32
        if gs:   # (sum, sumsq) per (image, group of 32) of the produced output, every chunk and pass included
            v = out.to(F64).reshape(b, c.ho * c.wo, c.cout // gs, gs).transpose(1, 2).reshape(b, c.cout // gs, -1)
            sums = torch.stack([v.sum(-1), (v * v).sum(-1)], -1) + STATS_PREFILL
            assert torch.allclose(st, sums, rtol=1e-5, atol=1e-3), float((st - sums).abs().max())
        assert torch.equal(out.view(torch.int32), out2.view(torch.int32)), "two runs differ"


@pytest.mark.parametrize("case", _cases(DGRAD_LAYERS), ids=_id)
def test_dgrad_against_float64(case):
    dev = _dev()
    name, (b, h, w) = case
    c = _Case(name, b, h, w, 202 + b + h + w, dev)
    c.gy[..., c.cout:] = 0   # the executors' gradients carry zero padding channels
    g_op = c.gy_operand()
    ref, ref16 = c.dgrad_ref(False), c.dgrad_ref(True)
    for k, (_, real, off) in enumerate(c.srcs):
        n = b * h * w * real
        runs = []
        for run in range(2):
            buf = torch.full((n + 64,), float("nan"), device=dev)
            buf[n:] = 7.0    # guard floats behind the output
            out = buf[:n].view(b, h, w, real)
            c.layer.dgrad(c.packed, k, g_op, b, h, w, out)
            runs.append(buf)
        pre = torch.randn(b, h, w, real, device=dev, generator=c.gen)
        acc = pre.clone()
        c.layer.dgrad(c.packed, k, g_op, b, h, w, acc, accumulate=True)
        torch.cuda.synchronize()
        got = runs[0][:n].view(b, h, w, real)
        want, want16 = ref[..., off:off + real], ref16[..., off:off + real]
        e16, e32 = _rel(got, want16), _rel(got, want)
        ea = _rel(acc.to(F64) - pre.to(F64), want16)
        print(f"{name} B={b} {h}x{w} source {k}: dgrad rel RMS vs fp16 operands {e16:.2e}, vs exact {e32:.2e}; accumulated {ea:.2e}")
        assert torch.isfinite(got).all() and torch.equal(runs[0][n:], torch.full((64,), 7.0, device=dev)), "wrote outside its source"
        assert e16 < FP16_TOL and e32 < FP32_TOL, (e16, e32)
        assert ea < FP16_TOL, ea
        assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32)), "two runs differ"


def _wgrad_cases():
    return _cases(list(LAYERS)) + [("c128", (32, 64, 64))]   # 32 x 64 x 64: several tiles per CTA in every block


@pytest.mark.parametrize("case", _wgrad_cases(), ids=_id)
def test_wgrad_against_float64(case):
    dev = _dev()
    from diamond_b200 import ops

    name, (b, h, w) = case
    c = _Case(name, b, h, w, 303 + b + h + w, dev)
    if b * (h + 1) * (w + 1) >= 2 * 128 * torch.cuda.get_device_properties(dev).multi_processor_count:
        print(f"{name} B={b} {h}x{w}: every CTA of a block runs two tiles or more")
    g_op = c.gy_operand(8.0)                         # the loss-scaled gradient ...
    inv = torch.tensor([0.125], device=dev)          # ... and its inverse scale
    ref, ref16 = c.wgrad_ref(False), c.wgrad_ref(True)
    taps = c.k * c.k
    pre = 0.5 * torch.randn(c.cout, c.cin_real, taps, device=dev, generator=c.gen)
    partial = torch.empty(_lib.lib().dmd_wgrad_partial_bytes(), dtype=torch.uint8, device=dev)
    for k, (stored, real, off) in enumerate(c.srcs):
        act_op = ops.prep_act(c.source(k))[0]
        dws = []
        for run in range(2):
            dw = pre.clone()
            c.layer.wgrad(g_op, act_op, stored, real, off, b, h, w, dw, inv, partial)
            dws.append(dw)
        torch.cuda.synchronize()
        dw = dws[0]
        got = dw[:, off:off + real].to(F64) - pre[:, off:off + real].to(F64)
        e16, e32 = _rel(got, ref16[:, off:off + real]), _rel(got, ref[:, off:off + real])
        print(f"{name} B={b} {h}x{w} source {k}: wgrad rel RMS vs fp16 operands {e16:.2e}, vs exact {e32:.2e}")
        assert e16 < FP16_TOL and e32 < FP32_TOL, (e16, e32)
        rest = torch.ones(c.cin_real, dtype=torch.bool, device=dev)
        rest[off:off + real] = False
        assert torch.equal(dw[:, rest].view(torch.int32), pre[:, rest].view(torch.int32)), "changed the other source's columns"
        assert torch.equal(dws[0].view(torch.int32), dws[1].view(torch.int32)), "two runs differ"


def test_wgrad_refuses_a_short_partial_buffer():
    dev = _dev()
    c = _Case("c128", 1, 8, 8, 1, dev)
    dw = torch.zeros(128, 128, 9, device=dev)
    short = torch.empty(1024, dtype=torch.uint8, device=dev)
    with pytest.raises(RuntimeError, match="partial buffer too small"):
        c.layer.wgrad(c.gy_operand(), c.gy_operand(), 128, 128, 0, 1, 8, 8, dw, None, short)
