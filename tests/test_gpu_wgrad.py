"""GPU: wgmma weight-gradient kernel (diamond_b200/csrc/wgrad_tc.cuh) and the dgrad packing helper against torch
autograd's conv2d_weight / conv2d_input (the reference's backward: nn.Conv2d under loss.backward(), blocks.py:18-19,96,109).

Operands are fp16 (PLC16), accumulation fp32: compared (a) with an fp16-operand fp64 reference to 2e-5 and (b) with exact
fp32 autograd to 2e-3 (the operand rounding itself)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-20))


def _h(t):
    return t.half().float()


def _wgrad_case(dev, b, h, w, cin, cout, taps, seed, stride=1):
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(seed)
    k = 3 if taps == 9 else 1
    x = torch.randn(b, cin, h, w, generator=g)
    ho, wo = h // stride, w // stride
    gy = torch.randn(b, cout, ho, wo, generator=g)
    wt = torch.zeros(cout, cin, k, k, requires_grad=True)
    y = F.conv2d(x, wt, stride=stride, padding=k // 2)
    (gw,) = torch.autograd.grad(y, wt, gy)
    yh = F.conv2d(_h(x).double(), wt.double(), stride=stride, padding=k // 2)
    (gw16,) = torch.autograd.grad(yh, wt, _h(gy).double())
    xn = ops.nchw_to_nhwc(x.to(dev), ops.round_up(cin, 8))
    gn = ops.nchw_to_nhwc(gy.to(dev), ops.round_up(cout, 8))
    x_op = ops.prep_act(xn)[0]
    g_op = ops.prep_act(gn, upsample=2 if stride == 2 else False)[0]     # stride 2: zero-inserted gradient at the input size
    dw = ops.conv2d_wgrad(g_op, ops.round_up(cout, 16), x_op, ops.round_up(cin, 16), b, h, w, cout, cin, taps)
    torch.cuda.synchronize()
    return dw.reshape(cout, cin, k, k).cpu(), gw16.float(), gw.detach()


@pytest.mark.parametrize("b,h,w,cin,cout,taps,stride", [
    (2, 16, 16, 64, 64, 9, 1),      # 8 tiles... multi-tile, one image row per ~8 tiles
    (3, 32, 32, 64, 64, 9, 1),      # ResBlock conv at 32x32
    (5, 64, 64, 64, 64, 9, 1),      # 64x64: 165 tiles > 132 CTAs (uneven tile ranges)
    (2, 8, 8, 64, 64, 9, 1),        # fewer tiles than SMs
    (2, 32, 32, 32, 64, 9, 1),      # Cin 32 (small config / actor-critic)
    (2, 32, 32, 64, 32, 9, 1),      # Cout 32: zero row groups
    (2, 64, 64, 15, 64, 9, 1),      # conv_in: 15 real input channels in a 16-channel operand
    (2, 64, 64, 64, 3, 9, 1),       # conv_out: 3 real output channels
    (2, 32, 32, 64, 64, 1, 1),      # 1x1 (skip projection / attention projections)
    (2, 32, 32, 64, 64, 9, 2),      # Downsample (stride 2): zero-inserted gradient
])
def test_wgrad_matches_autograd(b, h, w, cin, cout, taps, stride):
    dev = _dev()
    got, ref16, ref = _wgrad_case(dev, b, h, w, cin, cout, taps, 17 + cin + cout + taps, stride)
    e16, e32 = _rel(got, ref16), _rel(got, ref)
    print(f"wgrad B={b} {h}x{w} {cin}->{cout} taps={taps} s={stride}: err vs fp16-operand ref {e16:.2e}, vs fp32 autograd {e32:.2e}")
    assert e16 < 2e-5, e16
    assert e32 < 2e-3, e32


@pytest.mark.parametrize("b,h,w", [(32, 64, 64), (512, 8, 8), (16, 152, 280)], ids=["32x64x64", "512x8x8", "16x152x280"])
def test_wgrad_many_tiles_per_cta(b, h, w):
    """The persistent schedule at several tiles per CTA (the grid is min(tiles, SMs)): every CTA's partial sum covers a range
    of tiles, images straddle tiles (8x8) and the rows are wide (the 280-column CSGO frame).  Against the fp16-operand float64
    reference with the 2e-5 relative-RMS bound of test_wgrad_matches_autograd (measured, not derived), and two launches are
    bit-identical (the partials are reduced in a fixed order)."""
    dev = _dev()
    from diamond_b200 import ops

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tiles = -(-b * (h + 1) * (w + 1) // 128)
    assert tiles >= 2 * sms, (tiles, sms)      # every CTA runs two tiles or more
    g = torch.Generator(device=dev).manual_seed(b + h + w)
    x = torch.randn(b, 64, h, w, device=dev, generator=g)
    gy = torch.randn(b, 64, h, w, device=dev, generator=g)
    x_op = ops.prep_act(ops.nchw_to_nhwc(x))[0]
    g_op = ops.prep_act(ops.nchw_to_nhwc(gy))[0]
    dw = ops.conv2d_wgrad(g_op, 64, x_op, 64, b, h, w, 64, 64, 9)
    dw2 = ops.conv2d_wgrad(g_op, 64, x_op, 64, b, h, w, 64, 64, 9)
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_weight(_h(x).double(), (64, 64, 3, 3), _h(gy).double(), padding=1)
    e16 = _rel(dw.reshape(64, 64, 3, 3).double(), ref)
    print(f"wgrad B={b} {h}x{w}: {tiles} tiles on {sms} SMs, err vs fp16-operand ref {e16:.2e}")
    assert e16 < 2e-5, e16
    assert torch.equal(dw, dw2)


def test_wgrad_concat_halves_scale_and_accumulate():
    """A channel-concat conv (blocks.py:174) takes its weight gradient as two launches writing disjoint Cin ranges; inv_scale
    undoes the loss scale; accumulate adds to an existing gradient; two runs are bit-identical (fixed-order reduction)."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(5)
    b, h, w = 2, 16, 16
    x = torch.randn(b, 128, h, w, generator=g)
    gy = torch.randn(b, 64, h, w, generator=g)
    wt = torch.zeros(64, 128, 3, 3, requires_grad=True)
    (gw,) = torch.autograd.grad(F.conv2d(_h(x).double(), wt.double(), padding=1), wt, _h(gy * 8).double() / 8)
    g_op = ops.prep_act(ops.nchw_to_nhwc((gy * 8).to(dev)))[0]
    inv = torch.tensor([0.125], device=dev)
    dw = torch.full((64, 128, 9), 1.0, device=dev)
    for k in range(2):
        x_op = ops.prep_act(ops.nchw_to_nhwc(x[:, 64 * k:64 * (k + 1)].contiguous().to(dev)))[0]
        ops.conv2d_wgrad(g_op, 64, x_op, 64, b, h, w, 64, 64, 9, dw=dw, cin_tot=128, ci_off=64 * k, inv_scale=inv, accumulate=True)
    got = dw.reshape(64, 128, 3, 3).cpu() - 1.0
    assert _rel(got, gw.float()) < 2e-5
    dw2 = torch.full((64, 128, 9), 1.0, device=dev)
    for k in range(2):
        x_op = ops.prep_act(ops.nchw_to_nhwc(x[:, 64 * k:64 * (k + 1)].contiguous().to(dev)))[0]
        ops.conv2d_wgrad(g_op, 64, x_op, 64, b, h, w, 64, 64, 9, dw=dw2, cin_tot=128, ci_off=64 * k, inv_scale=inv, accumulate=True)
    assert torch.equal(dw, dw2)


@pytest.mark.parametrize("cin_tot,ci_off,cin_k,cout,taps", [(64, 0, 64, 64, 9), (128, 64, 64, 64, 9), (128, 0, 64, 64, 1), (64, 0, 64, 3, 9), (96, 64, 32, 32, 9)])
def test_dgrad_with_packed_transposed_weights(cin_tot, ci_off, cin_k, cout, taps):
    """dmd_pack_conv_weight_dgrad + dmd_conv2d_fprop on dL/dy == autograd's conv2d_input restricted to input channels
    [ci_off, ci_off + cin_k) (one launch per source of a concat)."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(23)
    b, h, w = 2, 16, 16
    k = 3 if taps == 9 else 1
    x = torch.zeros(b, cin_tot, h, w, requires_grad=True)
    wt = torch.randn(cout, cin_tot, k, k, generator=g) / math.sqrt(cin_tot * taps)
    gy = torch.randn(b, cout, h, w, generator=g)
    (gx,) = torch.autograd.grad(F.conv2d(x.double(), _h(wt).double(), padding=k // 2), x, _h(gy).double())
    ref = gx[:, ci_off:ci_off + cin_k].float()
    wpk, cin_p, cout_p = ops.pack_conv_weight_T(wt.to(dev), ci_off, cin_k)
    gn = ops.nchw_to_nhwc(gy.to(dev), ops.round_up(cout, 8))
    out, _ = ops.conv2d_fprop(gn, wpk, cin_k, cout_p, cin_p, taps)
    got = ops.nhwc_to_nchw(out).cpu()
    assert got.shape == ref.shape
    assert _rel(got, ref) < 2e-5, _rel(got, ref)
