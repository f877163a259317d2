"""CPU: shape validation, error behaviour and launch planning of the conv / prep entry points, through the host-only
C-ABI twins dmd_conv_plan / dmd_prep_plan (same code path as dmd_conv2d_fprop / dmd_prep_act up to the launch).  Pointers
are dummies: the plan functions only test them for NULL."""
import ctypes as C

import pytest

from diamond_b200 import _lib

P = 0x1000  # any non-null address


def _conv(**kw):
    d = _lib.ConvDesc()
    base = dict(src0=P, out=P, wpk=P, C0=64, C1=0, B=32, H=64, W=64, taps=9, stride=1, Cout=64, CoutPad=64)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    info = _lib.ConvPlanInfo()
    rc = _lib.lib().dmd_conv_plan(C.byref(d), C.byref(info))
    return rc, info, _lib.lib().dmd_last_error().decode()


def _prep(**kw):
    d = _lib.PrepDesc()
    base = dict(src0=P, dst0=P, C0=64, C1=0, B=32, Hs=64, Ws=64, mode=0)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    blocks, ppb, nsrc = C.c_int(), C.c_int(), C.c_int()
    rc = _lib.lib().dmd_prep_plan(C.byref(d), C.byref(blocks), C.byref(ppb), C.byref(nsrc))
    return rc, blocks.value, ppb.value, nsrc.value, _lib.lib().dmd_last_error().decode()


def test_dominant_conv_plan():
    """3x3 64->64 @64x64, 32 images (SURVEY.md Appendix A row 2): positions = 32*65*65 on the padded line."""
    rc, i, _ = _conv()
    assert rc == 0
    assert i.tiles == -(-32 * 65 * 65 // 128) == 1057
    assert i.kslabs == 4 and i.acc_cols == 64
    assert i.stages == 16      # direct epilogue (no staging tile): four tiles' worth of 8.2 KB slabs next to 72 KB of weights
    assert i.weight_bytes == 9 * 64 * 64 * 2
    assert i.smem_bytes <= 227 * 1024


@pytest.mark.parametrize("kw,kslabs,cols", [
    (dict(C0=64, C1=64, src1=P), 8, 64),                                              # u-block conv1: x || skip
    (dict(C0=16, precise=1, src0_lo=P), 3, 64),                                       # conv_in, split-fp16
    (dict(C0=64, Cout=3, CoutPad=16), 4, 16),                                         # conv_out
    (dict(C0=64, xsrc0=P, xsrc0_lo=P, xsrc1=P, xsrc1_lo=P, xC0=64, xC1=64, wpk_x=P), 4 + 16, 64),  # conv2 + fused projection: hi and lo slabs once each (24 MMAs)
    (dict(C0=64, taps=1), 4, 64),
    (dict(C0=64, CoutPad=128, Cout=128, H=32, W=32), 4, 128),                         # 147 KB of weights: narrow images only
    (dict(Cout=48, CoutPad=48, H=32, W=32), 4, 64),                                   # CoutPad below the accumulator width
    (dict(Cout=96, CoutPad=96, H=16, W=24), 4, 128),
    (dict(C0=128, H=32, W=32), 8, 64),                                                # one 128-channel source
])
def test_conv_plan_variants(kw, kslabs, cols):
    rc, i, err = _conv(**kw)
    assert rc == 0, err
    assert i.kslabs == kslabs and i.acc_cols == cols
    assert 2 <= i.stages <= 24 and i.smem_bytes <= 227 * 1024


@pytest.mark.parametrize("hw,tiles", [(32, -(-32 * 33 * 33 // 128)), (16, -(-32 * 17 * 17 // 128)), (8, -(-32 * 81 // 128))])
def test_conv_tiles_per_level(hw, tiles):
    rc, i, _ = _conv(H=hw, W=hw)
    assert rc == 0 and i.tiles == tiles


@pytest.mark.parametrize("kw,needle", [
    (dict(taps=4), "taps must be 1 or 9"),
    (dict(stride=3), "stride must be 1 or 2"),
    (dict(C0=24), "multiples of 16"),
    (dict(C0=128, C1=64, src1=P), "multiples of 16, total <="),
    (dict(C1=64), "src1/C1 mismatch"),
    (dict(precise=1), "low operand parts"),
    (dict(CoutPad=72), "bad Cout"),
    (dict(Cout=80), "bad Cout"),
    (dict(stride=2, H=63), "stride 2 needs even"),
    (dict(out_stats=P, out_gs=32, Cout=48, CoutPad=48), "out_stats needs Cout"),
    (dict(out_stats=P, out_gs=24), "out_gs must be"),
    (dict(out_stats=P, out_gs=32, H=4, W=4), "image too small"),
    (dict(C0=64, C1=64, src1=P, W=600, H=8, B=1), "shared memory too small"),
    (dict(src0=0), "null src0/out/wpk"),
    (dict(wpk_x=P), "bad fused projection operands"),
    (dict(debug=1), "debug / debug_buf must be 0"),
])
def test_conv_rejections_fail_loudly(kw, needle):
    rc, _, err = _conv(**kw)
    assert rc != 0 and needle in err, err


@pytest.mark.parametrize("kw,w_ok,w_bad", [
    (dict(), 1160, 1168),                                        # 64 -> 64: 72 KB of weights
    (dict(C0=64, C1=64, src1=P), 584, 592),                      # 128 -> 64: 144 KB of weights
    (dict(Cout=128, CoutPad=128), 584, 592),                     # 64 -> 128: 144 KB of weights
])
def test_width_limit_is_the_shared_memory_ring(kw, w_ok, w_bad):
    """The halo slab is 32*(128 + 2*(W+2)) bytes and two of them must fit next to the resident weights (the direct epilogue
    needs no staging tile); wider images are rejected (config-5 shapes need a strip path, DESIGN.md section 6)."""
    rc, i, err = _conv(B=1, H=8, W=w_ok, **kw)
    assert rc == 0 and i.stages >= 2, err
    rc, _, err = _conv(B=1, H=8, W=w_bad, **kw)
    assert rc != 0 and "shared memory too small" in err


def test_prep_plan_block_granularity():
    """Low-resolution levels get smaller blocks so that the grid still covers the 132 SMs (>= 264 blocks wanted)."""
    rc, blocks, ppb, nsrc, _ = _prep()
    assert rc == 0 and ppb == 256 and nsrc == 1 and blocks >= 264
    rc, blocks, ppb, nsrc, _ = _prep(Hs=16, Ws=16)
    assert rc == 0 and ppb == 64
    rc, blocks, ppb, nsrc, _ = _prep(Hs=32, Ws=32, C1=64, src1=P, dst1=P)
    assert rc == 0 and nsrc == 2
    # the widest norm the executors build: 4 groups of 32 in each source of an up-path concat
    rc, *_, err = _prep(Hs=32, Ws=32, mode=1, silu=1, stats0=P, gs0=32, film=P, C0=128, C1=128, src1=P, dst1=P, stats1=P, gs1=32)
    assert rc == 0, err


@pytest.mark.parametrize("kw,needle", [
    (dict(C0=12), "multiples of 8"),
    (dict(mode=3), "bad mode"),
    (dict(mode=1), "needs stats0"),
    (dict(mode=1, stats0=P, gs0=32), "needs film"),
    (dict(mode=2, stats0=P, gs0=32), "needs gamma/beta"),
    (dict(mode=1, stats0=P, gs0=32, film=P, upsample=1), "norm + upsample unsupported"),
    (dict(Hs=2, Ws=2), "image too small"),
    (dict(C1=64), "src1/dst1/C1 mismatch"),
    (dict(dst0=0), "null src0/dst0"),
])
def test_prep_rejections_fail_loudly(kw, needle):
    rc, *_, err = _prep(**kw)
    assert rc != 0 and needle in err, err


@pytest.mark.parametrize("kw,needle", [
    (dict(C0=15), "multiples of 8"),                        # 15 image channels are zero-padded to 16 before the prep
    # both prep kernels keep (mean, rstd) of at most 4 groups per source in shared memory: source 0 and source 1
    (dict(mode=1, stats0=P, gs0=8, film=P), "at most 4 groups per source"),
    (dict(mode=1, stats0=P, gs0=32, film=P, C1=64, src1=P, dst1=P, stats1=P, gs1=8), "at most 4 groups per source"),
    (dict(mode=2, stats0=P, gs0=32, gamma=P, beta=P, C0=32, C1=128, src1=P, dst1=P, stats1=P, gs1=16), "at most 4 groups per source"),
], ids=["c15", "groups-src0", "groups-src1-ada", "groups-src1-gn"])
def test_prep_channel_and_group_limits(kw, needle):
    rc, *_, err = _prep(**kw)
    assert rc != 0 and needle in err, err
