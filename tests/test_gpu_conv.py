"""GPU: wgmma conv kernel (C-ABI dmd_conv2d_fprop) vs torch fp32 reference ops of the same op.

Operands are rounded to fp16 inside the kernel (fp32 accumulate), so the reference is evaluated both with exact fp32
operands (tolerance 2e-3 of the output rms: the TF32-class error the reference's own GPU path has, trainer.py:41) and
with fp16-rounded operands (tolerance 2e-5: only accumulation order differs)."""
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
    return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-12))


def _h(x):
    return x.half().float()


def _run_conv(dev, b, h, w, c0, c1, cout, taps=9, upsample=False, stride=1, prologue=0, silu=False, residual=False,
              want_stats=False, seed=0, debug=0, precise=False, trs=False):
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(seed)
    k = 3 if taps == 9 else 1
    cin = c0 + c1
    x0 = torch.randn(b, c0, h, w, generator=g)
    x1 = torch.randn(b, c1, h, w, generator=g) * 1.5 + 0.3 if c1 else None
    wt = torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)
    bias = torch.randn(cout, generator=g) * 0.1
    xin = torch.cat([x0, x1], 1) if c1 else x0
    gs = 32 if cin % 32 == 0 else cin
    film = gamma = beta = None
    pre = xin
    if prologue == 1:
        film_full = torch.randn(b, 2 * cin + 5, generator=g) * 0.3
        scale, shift = film_full[:, 5:5 + cin], film_full[:, 5 + cin:5 + 2 * cin]
        pre = F.group_norm(xin, cin // gs, eps=1e-5) * (1 + scale[:, :, None, None]) + shift[:, :, None, None]
        film = film_full
    elif prologue == 2:
        gamma = 1 + 0.2 * torch.randn(cin, generator=g)
        beta = 0.1 * torch.randn(cin, generator=g)
        pre = F.group_norm(xin, cin // gs, gamma, beta, eps=1e-5)
    if silu:
        pre = F.silu(pre)
    if upsample:
        pre = F.interpolate(pre, scale_factor=2.0, mode="nearest")
    ho, wo = pre.shape[2] // stride, pre.shape[3] // stride
    res = torch.randn(b, cout, ho, wo, generator=g) if residual else None
    ref32 = F.conv2d(pre, wt, bias, stride=stride, padding=k // 2)
    ref16 = F.conv2d(_h(pre).double(), _h(wt).double(), bias.double(), stride=stride, padding=k // 2).float()
    if residual:
        ref32, ref16 = ref32 + res, ref16 + res

    cin_pad = ops.round_up(cin, 16)
    c0s = ops.round_up(c0, 8)
    s0 = ops.nchw_to_nhwc(x0.to(dev), c0s)
    s1 = ops.nchw_to_nhwc(x1.to(dev)) if c1 else None
    cin_pad = ops.round_up(c0s, 16) + (ops.round_up(c1, 16) if c1 else 0)
    wpk, cout_pad = ops.pack_conv_weight(wt.to(dev), cin_pad, c0_real=c0, c0_store=ops.round_up(c0s, 16), precise=precise, trs=trs)
    kw = {}
    if prologue:
        gs0 = gs if c0 % gs == 0 else c0
        kw.update(stats0=ops.gn_stats(s0, gs0), gs0=gs0)
        if c1:
            kw.update(stats1=ops.gn_stats(s1, gs), gs1=gs)
    out, st = ops.conv2d_fprop(
        s0, wpk, cout, cout_pad, cin_pad, taps, src1=s1, bias=bias.to(dev), upsample=upsample, stride=stride,
        prologue=prologue, silu=silu, film=film.to(dev) if film is not None else None, film_off=5,
        gamma=gamma.to(dev) if gamma is not None else None, beta=beta.to(dev) if beta is not None else None,
        residual=ops.nchw_to_nhwc(res.to(dev)) if residual else None,
        out_gs=(32 if cout % 32 == 0 else 0) if want_stats else 0, debug=debug, precise=precise, trs=trs, **kw)
    got = ops.nhwc_to_nchw(out).cpu()
    torch.cuda.synchronize()
    return got, ref32, ref16, (st.cpu() if st is not None else None)


CASES = [
    dict(b=2, h=64, w=64, c0=64, c1=0, cout=64),                                    # d0 conv (Appendix A row 2)
    dict(b=3, h=32, w=32, c0=64, c1=64, cout=64),                                   # u2.conv1 two-source
    dict(b=2, h=64, w=64, c0=64, c1=64, cout=64, taps=1),                           # u3.proj 1x1
    dict(b=2, h=64, w=64, c0=15, c1=0, cout=64),                                    # conv_in (15 -> pad 16)
    dict(b=2, h=64, w=64, c0=64, c1=0, cout=3),                                     # conv_out (Cout 3)
    dict(b=2, h=64, w=64, c0=64, c1=0, cout=64, stride=2),                          # downsamples.1
    dict(b=2, h=16, w=16, c0=64, c1=0, cout=64, upsample=True),                     # upsamples
    dict(b=5, h=8, w=8, c0=64, c1=0, cout=64),                                      # 8x8 level, tile spans images
    dict(b=1, h=8, w=8, c0=64, c1=64, cout=64),                                     # single small image (partial tile)
    dict(b=2, h=32, w=32, c0=32, c1=64, cout=64),                                   # Cin 96 (generic chunk count)
    dict(b=2, h=64, w=64, c0=3, c1=0, cout=32),                                     # actor-critic stem 3 -> 32
    dict(b=2, h=24, w=40, c0=32, c1=0, cout=32),                                    # non-square, non power of two
    dict(b=2, h=32, w=32, c0=64, c1=0, cout=48),                                    # CoutPad 48 < 64 accumulator columns
    dict(b=3, h=16, w=24, c0=64, c1=0, cout=96),                                    # CoutPad 96 < 128 accumulator columns
    dict(b=2, h=32, w=32, c0=64, c1=0, cout=128),                                   # the 128-column kernel (narrow images)
    dict(b=2, h=32, w=32, c0=64, c1=0, cout=128, taps=1),
    dict(b=2, h=32, w=32, c0=128, c1=0, cout=64),                                   # one 128-channel source (16 prep chunks)
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_conv_plain(case):
    dev = _dev()
    got, ref32, ref16, _ = _run_conv(dev, **case)
    assert got.shape == ref32.shape
    assert _rel(got, ref16) < 2e-5, ("fp16-operand reference", _rel(got, ref16))
    assert _rel(got, ref32) < 2e-3, ("fp32 reference", _rel(got, ref32))


# row-stacked weights hold 3 * CoutPad columns, at most 256 (CoutPad <= 80)
@pytest.mark.parametrize("case", [c for c in CASES if c.get("taps", 9) == 9 and c["cout"] <= 80],
                         ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_conv_row_stacked_taps(case):
    """The tap-row-stacked weight layout of the 3x3 convs (the three taps of a kernel row side by side, N = 3 * Cout; the kernel
    addresses each tap inside its row, conv_tc.cuh) -- same results as the tap-major layout."""
    dev = _dev()
    got, ref32, ref16, _ = _run_conv(dev, trs=True, **case)
    assert got.shape == ref32.shape
    assert _rel(got, ref16) < 2e-5, ("fp16-operand reference", _rel(got, ref16))
    assert _rel(got, ref32) < 2e-3, ("fp32 reference", _rel(got, ref32))


@pytest.mark.parametrize("shape", [dict(b=2, h=64, w=64, c0=64, c1=0, cout=64), dict(b=3, h=16, w=16, c0=64, c1=64, cout=64),
                                   dict(b=4, h=8, w=8, c0=64, c1=0, cout=64), dict(b=32, h=64, w=64, c0=64, c1=0, cout=64)],
                         ids=["64x64", "16x16cat", "8x8", "bench"])
def test_conv_row_stacked_norm_prologue_residual_stats(shape):
    dev = _dev()
    got, ref32, _, st = _run_conv(dev, prologue=1, silu=True, residual=True, want_stats=True, seed=3, trs=True, **shape)
    assert _rel(got, ref32) < 2e-3, _rel(got, ref32)
    b, c, h, w = got.shape
    v = got.double().reshape(b, c // 32, 32 * h * w)
    want = torch.stack([v.sum(-1), (v * v).sum(-1)], -1)
    assert torch.allclose(st, want, rtol=1e-5, atol=1e-3), float((st - want).abs().max())


@pytest.mark.parametrize("prologue,silu", [(1, True), (2, True), (1, False)])
@pytest.mark.parametrize("shape", [dict(b=2, h=64, w=64, c0=64, c1=0, cout=64), dict(b=3, h=16, w=16, c0=64, c1=64, cout=64),
                                   dict(b=4, h=8, w=8, c0=64, c1=0, cout=64), dict(b=2, h=32, w=32, c0=128, c1=0, cout=64),
                                   dict(b=2, h=16, w=16, c0=64, c1=0, cout=128)],
                         ids=["64x64", "16x16cat", "8x8", "32x32c128", "16x16cout128"])
def test_conv_fused_norm_prologue_residual_stats(prologue, silu, shape):
    dev = _dev()
    got, ref32, _, st = _run_conv(dev, prologue=prologue, silu=silu, residual=True, want_stats=True, seed=3, **shape)
    assert _rel(got, ref32) < 2e-3, _rel(got, ref32)
    # epilogue GroupNorm partials == sums over the produced tensor
    b, c, h, w = got.shape
    v = got.double().reshape(b, c // 32, 32 * h * w)
    want = torch.stack([v.sum(-1), (v * v).sum(-1)], -1)
    assert torch.allclose(st, want, rtol=1e-5, atol=1e-3), float((st - want).abs().max())


@pytest.mark.parametrize("case", [
    dict(b=2, h=64, w=64, c0=64, c1=64, cout=64, taps=1),                    # u3.proj: raw residual stream, two sources
    dict(b=2, h=64, w=64, c0=15, c1=0, cout=64),                             # conv_in
    dict(b=2, h=64, w=64, c0=64, c1=0, cout=3, prologue=2, silu=True),       # conv_out(silu(norm_out(x)))
    dict(b=3, h=16, w=16, c0=32, c1=64, cout=64, taps=1),                    # proj with unequal sources
], ids=["proj", "conv_in", "conv_out", "proj96"])
def test_conv_precise_split_fp16(case):
    """split-fp16 (A_hi W_hi + A_lo W_hi + A_hi W_lo): the layers that feed the residual stream directly match the fp32
    reference to ~1e-6 instead of the 4e-4 of single fp16 operands."""
    dev = _dev()
    got, ref32, _, _ = _run_conv(dev, precise=True, seed=5, **case)
    assert _rel(got, ref32) < 5e-6, _rel(got, ref32)


@pytest.mark.parametrize("trs", [False, True], ids=["tap-major", "row-stacked"])
def test_conv_with_fused_skip_projection(trs):
    """ResBlock tail (blocks.py:142-145): conv2(silu(norm2(t))) + proj(cat(x, skip)) in ONE launch — the 1x1 projection is
    extra K (split-fp16, centre tap) accumulated into the same accumulator tile."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(11)
    b, h, w = 3, 32, 32
    t = torch.randn(b, 64, h, w, generator=g)
    x, sk = torch.randn(b, 64, h, w, generator=g) * 2, torch.randn(b, 64, h, w, generator=g) + 0.5
    w2 = torch.randn(64, 64, 3, 3, generator=g) / 24; b2 = torch.randn(64, generator=g) * 0.1
    wp = torch.randn(64, 128, 1, 1, generator=g) / 11; bp = torch.randn(64, generator=g) * 0.1
    ref = F.conv2d(_h(t).double(), _h(w2).double(), b2.double(), padding=1).float() + F.conv2d(torch.cat([x, sk], 1), wp, bp)
    tn, xn, sn = (ops.nchw_to_nhwc(v.to(dev)) for v in (t, x, sk))
    n0 = ops.prep_act(tn)[0]
    res = ops.prep_act(xn, src1=sn, also_raw=False, split=True)  # raw mode: main operand = raw hi, lo parts via split
    xh0, xh1, xl0, xl1 = res[0], res[1], res[6], res[7]
    wpk2, cp = ops.pack_conv_weight(w2.to(dev), 64, trs=trs)
    wpkx, _ = ops.pack_conv_weight(wp.to(dev), 128, precise=True)
    out, _ = ops.conv2d_operand(n0, None, 64, 0, b, h, w, wpk2, 64, cp, bias=b2.to(dev),
                                xproj=(xh0, xh1, xl0, xl1, 64, 64, wpkx, bp.to(dev)), trs=trs)
    got = ops.nhwc_to_nchw(out).cpu()
    assert _rel(got, ref) < 2e-5, _rel(got, ref)


@pytest.mark.parametrize("cin,cout", [(64, 64), (32, 64), (64, 128)])
def test_conv_dgrad_is_the_forward_kernel_with_transposed_flipped_weights(cin, cout):
    """Building block of the training rows (SURVEY.md 8 a18): backward-data of a 3x3 / stride-1 / pad-1 convolution
    (every ResBlock conv, blocks.py:137-139) is the SAME implicit GEMM on the output gradient with the weights transposed
    (Cin <-> Cout) and the taps flipped, so it runs on the wgmma kernel unchanged.  Checked against torch autograd."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(11)
    b, h, w = 2, 32, 32
    x = torch.randn(b, cin, h, w, generator=g, requires_grad=True)
    wt = torch.randn(cout, cin, 3, 3, generator=g) / math.sqrt(cin * 9)
    gy = torch.randn(b, cout, h, w, generator=g)
    (gx,) = torch.autograd.grad(F.conv2d(x, wt, padding=1), x, gy)
    wt_t = wt.transpose(0, 1).flip(2, 3).contiguous()            # [cin, cout, 3, 3]
    gx16 = F.conv2d(_h(gy).double(), _h(wt_t).double(), padding=1).float()
    assert _rel(gx16, gx) < 2e-3                                   # the identity itself (fp16 operands vs exact)
    wpk, cpad = ops.pack_conv_weight(wt_t.to(dev), cout)
    out, _ = ops.conv2d_fprop(ops.nchw_to_nhwc(gy.to(dev)), wpk, cin, cpad, cout, 9)
    got = ops.nhwc_to_nchw(out).cpu()
    assert got.shape == gx.shape
    assert _rel(got, gx16) < 2e-5, _rel(got, gx16)
    assert _rel(got, gx) < 2e-3, _rel(got, gx)


def test_conv_linearity_and_zero():
    """size-independent properties: conv(0)=bias, conv(a+b)-bias = (conv(a)-bias)+(conv(b)-bias) up to fp16 rounding."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(1)
    wt = torch.randn(64, 64, 3, 3, generator=g) / 24
    bias = torch.randn(64, generator=g)
    wpk, cp = ops.pack_conv_weight(wt.to(dev), 64)
    z = torch.zeros(2, 32, 32, 64, device=dev)
    out, _ = ops.conv2d_fprop(z, wpk, 64, cp, 64, bias=bias.to(dev))
    assert torch.equal(out.cpu(), bias.expand(2, 32, 32, 64))
    # exactly representable inputs -> fp16 rounding is exact -> integer-valued linearity holds to accumulate order
    a = torch.randint(-4, 5, (2, 32, 32, 64), generator=g).float().to(dev)
    bb = torch.randint(-4, 5, (2, 32, 32, 64), generator=g).float().to(dev)
    oa, _ = ops.conv2d_fprop(a, wpk, 64, cp, 64)
    ob, _ = ops.conv2d_fprop(bb, wpk, 64, cp, 64)
    oab, _ = ops.conv2d_fprop(a + bb, wpk, 64, cp, 64)
    assert torch.allclose(oab, oa + ob, atol=1e-4)


def test_attention_matches_torch():
    dev = _dev()
    from diamond_b200 import ops
    from oracle import torch_oracle as O

    g = torch.Generator().manual_seed(2)
    for c in (64, 32):
        x = torch.randn(3, c, 8, 8, generator=g) * 2 + 0.5
        sd = {
            "a.norm.norm.weight": 1 + 0.2 * torch.randn(c, generator=g), "a.norm.norm.bias": 0.1 * torch.randn(c, generator=g),
            "a.qkv_proj.weight": torch.randn(3 * c, c, 1, 1, generator=g) / math.sqrt(c), "a.qkv_proj.bias": 0.1 * torch.randn(3 * c, generator=g),
            "a.out_proj.weight": torch.randn(c, c, 1, 1, generator=g) / math.sqrt(c), "a.out_proj.bias": 0.1 * torch.randn(c, generator=g),
        }
        ref = O.self_attention(x, sd, "a.")
        xs = ops.nchw_to_nhwc(x.to(dev))
        gs = 32
        out, st = ops.attn_fwd(xs, ops.gn_stats(xs, gs), sd["a.norm.norm.weight"].to(dev), sd["a.norm.norm.bias"].to(dev),
                               sd["a.qkv_proj.weight"].reshape(3 * c, c).contiguous().to(dev), sd["a.qkv_proj.bias"].to(dev),
                               sd["a.out_proj.weight"].reshape(c, c).contiguous().to(dev), sd["a.out_proj.bias"].to(dev), gs)
        got = ops.nhwc_to_nchw(out).cpu()
        assert _rel(got, ref) < 1e-5, _rel(got, ref)
        v = got.double().reshape(3, c // gs, gs * 64)
        want = torch.stack([v.sum(-1), (v * v).sum(-1)], -1)
        assert torch.allclose(st.cpu(), want, rtol=1e-5, atol=1e-3)
