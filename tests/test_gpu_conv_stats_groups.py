"""GPU: the conv epilogue's GroupNorm partial sums for every output group size it accepts (16, 32, 64, 128 channels).

The epilogue compiles one statistics path per group size, so each size is checked on its own: the (sum, sumsq) per
(image, group) must equal float64 sums over the kernel's own fp32 output, for tiles inside one image and for tiles that
straddle images (8x8 images: 81 positions, a 128-row tile touches up to three)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


# at most 4 groups per image (the host rejects Cout / gs > 4)
CASES = [(cout, gs, b, hw) for cout, gs in [(16, 16), (32, 16), (64, 16), (64, 32), (64, 64), (128, 32), (128, 64), (128, 128)]
         for b, hw in [(3, 32), (5, 8)]]


@pytest.mark.parametrize("cout,gs,b,hw", CASES, ids=lambda v: str(v))
def test_conv_stats_per_group_size(cout, gs, b, hw):
    from diamond_b200 import ops

    dev = _dev()
    g = torch.Generator().manual_seed(cout * 1000 + gs + hw)
    cin = 64
    x = torch.randn(b, cin, hw, hw, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) / math.sqrt(cin * 9)
    # a per-channel offset makes the groups' sums clearly different, so a sum credited to the wrong group shows
    bias = torch.randn(cout, generator=g) * 0.1 + torch.arange(cout, dtype=torch.float32) * 0.05
    s0 = ops.nchw_to_nhwc(x.to(dev))
    wpk, cout_pad = ops.pack_conv_weight(wt.to(dev), cin)
    out, st = ops.conv2d_fprop(s0, wpk, cout, cout_pad, cin, 9, bias=bias.to(dev), out_gs=gs)
    torch.cuda.synchronize()
    o = out.double().cpu().reshape(b, hw * hw, cout // gs, gs)
    want = torch.stack([o.sum(dim=(1, 3)), o.pow(2).sum(dim=(1, 3))], dim=-1)
    got = st.cpu()
    assert got.shape == want.shape == (b, cout // gs, 2)
    # the error bound derived from the epilogue's fp32 addition chain and its fp64 atomics (test_gpu_conv_schedule.py): gamma_m
    # of the sum of |terms| with m counted over the tiles of a CTA
    from test_gpu_conv_schedule import stats_excess

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tiles = -(-b * (hw + 1) ** 2 // 128)
    tmax = -(-tiles // min(tiles, sms))
    err = stats_excess(st, out.view(b, hw, hw, cout), gs, tmax, hw, hw)
    assert err <= 1.0, err
