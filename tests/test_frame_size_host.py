"""CPU: what frame sizes beyond 64 x 64 need from the host side.  The oracle against the reference's own outputs at 84 x 84 and
150 x 280 (tests/golden/denoiser_84x84.npz, denoiser_150x280.npz; oracle/make_golden_frame_size.py), every conv of the
default net's 88 x 88 and 152 x 280 U-Net plans through the host-only planner, and the argument checks of the any-L attention
entry point (which run before any CUDA call)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from diamond_b200 import _lib
from oracle import torch_oracle as O
from oracle.make_golden_frame_size import FRAME_SIZE_CASES, initial_noise, noise_checksum

P = 0x1000  # any non-null address


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


@pytest.mark.parametrize("name", list(FRAME_SIZE_CASES))
def test_oracle_matches_reference_golden_at_frame_size(golden_dir, name):
    c = FRAME_SIZE_CASES[name]
    g = _load(golden_dir, name)
    inner = c["inner"]
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    cfg = O.DenoiserCfg(inner=inner)
    obs, act, x_noisy = O.synthetic_inputs(c["b"], inner, c["h"], c["w"], c["iseed"])
    b, t, ch, h, w = obs.shape
    sig = torch.from_numpy(g["sigmas_in"])
    with torch.no_grad():
        mo = O.model_output(x_noisy, sig, obs.reshape(b, t * ch, h, w), act, sd, cfg)
        dn = O.wrap_model_output(x_noisy, mo, sig, cfg)
    ref_mo = torch.from_numpy(g["model_output"])
    assert torch.allclose(mo, ref_mo, rtol=1e-5, atol=1e-5), float((mo - ref_mo).abs().max())
    ref_dn = torch.from_numpy(g["denoised"])
    assert float((dn != ref_dn).float().mean()) < 1e-3 and float((dn - ref_dn).abs().max()) <= 2 / 255 + 1e-6
    # the sampler: the whole trajectory where the fixture has it (84 x 84), the final frame of the 10 steps otherwise
    s = c["sampler"]
    assert torch.equal(O.build_sigmas(s.num_steps_denoising, s.sigma_min, s.sigma_max, s.rho), torch.from_numpy(g["sampler_sigmas"]))
    x0 = initial_noise(c)   # the reference's first draw; the 150 x 280 fixture stores only its checksum
    assert np.allclose(noise_checksum(x0), g["x0_checksum"], rtol=1e-12, atol=0)
    if "x0" in g:
        assert torch.equal(x0, torch.from_numpy(g["x0"]))
    with torch.no_grad():
        x, traj = O.sample(obs, act, x0, sd, cfg, s)
    if "trajectory" in g:
        diff = (torch.stack(traj) - torch.from_numpy(g["trajectory"])).abs()
        assert float((diff > 1e-4).float().mean()) < 2e-3, float(diff.max())
    diff = (x - torch.from_numpy(g["sample_x"])).abs()
    assert float((diff > 1e-4).float().mean()) < 2e-3, float(diff.max())


def test_frame_size_fixtures_fit_their_budget(golden_dir):
    sizes = [os.path.getsize(os.path.join(golden_dir, n + ".npz")) for n in FRAME_SIZE_CASES]
    assert max(sizes) < 1_000_000 and sum(sizes) <= 3 * 1024 * 1024, sizes


def _conv(**kw):
    d = _lib.ConvDesc()
    for k, v in {**dict(src0=P, out=P, wpk=P, C0=64, C1=0, taps=9, stride=1, Cout=64, CoutPad=64), **kw}.items():
        setattr(d, k, v)
    info = _lib.ConvPlanInfo()
    rc = _lib.lib().dmd_conv_plan(C.byref(d), C.byref(info))
    return rc, info, _lib.lib().dmd_last_error().decode()


def _default_net_convs(h, w, b):
    """Every distinct conv of the default net's plan (4 levels of 64 channels) at an h x w frame: conv_in and conv_out at
    h x w, everything else at the padded size and its halvings."""
    stats = dict(out_stats=P, out_gs=32)
    hp, wp = -(-h // 8) * 8, -(-w // 8) * 8
    yield "conv_in", dict(B=b, H=h, W=w, C0=16, precise=1, src0_lo=P)
    yield "conv_out", dict(B=b, H=h, W=w, Cout=3, CoutPad=16)
    for lv in range(4):
        H, W = hp >> lv, wp >> lv
        yield f"3x3+stats L{lv}", dict(B=b, H=H, W=W, **stats)
        yield f"skip concat L{lv}", dict(B=b, H=H, W=W, C1=64, src1=P, **stats)
        yield f"conv2+projection L{lv}", dict(B=b, H=H, W=W, xsrc0=P, xsrc0_lo=P, xsrc1=P, xsrc1_lo=P, xC0=64, xC1=64, wpk_x=P, **stats)
        if lv < 3:
            yield f"stride-2 down L{lv}", dict(B=b, H=H, W=W, stride=2, **stats)


@pytest.mark.parametrize("h,w", [(150, 280), (84, 84)])
@pytest.mark.parametrize("b", [1, 8, 64])
def test_every_conv_of_the_frame_size_plans_fits(h, w, b):
    for name, kw in _default_net_convs(h, w, b):
        rc, info, err = _conv(**kw)
        assert rc == 0, (name, err)
        assert info.stages >= 2 and info.smem_bytes <= 227 * 1024, (name, info.stages, info.smem_bytes)


def test_attn_scratch_bytes():
    lib = _lib.lib()
    assert lib.dmd_attn_scratch_bytes(8, 665, 64) == 8 * 665 * 3 * 64 * 4
    assert lib.dmd_attn_scratch_bytes(3, 121, 32) == 3 * 121 * 3 * 32 * 4
    assert lib.dmd_attn_scratch_bytes(8, 64, 64) == 0      # one launch, no scratch
    assert lib.dmd_attn_scratch_bytes(0, 665, 64) == 0


@pytest.mark.parametrize("kw,needle", [
    (dict(scratch_bytes=8 * 665 * 3 * 64 * 4 - 4), "scratch too small"),
    (dict(x=None), "bad arguments"),
    (dict(L=0), "bad arguments"),
])
def test_attn_scratch_entry_point_rejections(kw, needle):
    a = dict(x=P, L=665, scratch_bytes=0)
    a.update(kw)
    rc = _lib.lib().dmd_attn_fwd_scratch(a["x"], *[P] * 9, 8, a["L"], 64, 32, 1e-5, P, a["scratch_bytes"], None)
    err = _lib.lib().dmd_last_error().decode()
    assert rc != 0 and needle in err, err
