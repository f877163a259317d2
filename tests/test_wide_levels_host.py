"""CPU: nets with 128-channel levels.  The float32 oracle (oracle/torch_oracle.py) reproduces the reference's own outputs
for a [64, 128, 128, 128] denoiser and a [128] * 4 reward / termination model (tests/golden/*_wide.npz, written by
oracle/make_golden_wide.py), and the executors' create calls refuse levels wider than 128 channels, naming the limit,
before they touch a device."""
import os

import numpy as np
import pytest
import torch

from diamond_b200 import _lib


def _rel(a, b):
    return float((a - b).double().norm() / b.double().norm().clamp_min(1e-300))


def test_oracle_matches_wide_denoiser_golden(golden_dir):
    from oracle import torch_oracle as O
    from oracle.make_golden_wide import DENOISER_WIDE as c

    g = np.load(os.path.join(golden_dir, "denoiser_wide.npz"))
    inner = c["inner"]
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    obs, act, x_noisy = O.synthetic_inputs(c["b"], inner, c["h"], c["w"], c["iseed"])
    b, t, ch, h, w = obs.shape
    with torch.no_grad():
        mo = O.model_output(x_noisy, torch.from_numpy(g["sigmas_in"]), obs.reshape(b, t * ch, h, w), act, sd, O.DenoiserCfg(inner=inner))
    assert _rel(mo, torch.from_numpy(g["model_output"])) < 1e-5


def test_oracle_matches_wide_rew_end_golden(golden_dir):
    from oracle import torch_oracle as O
    from oracle.make_golden_wide import REW_END_WIDE as c

    g = np.load(os.path.join(golden_dir, "rew_end_wide.npz"))
    cfg = c["cfg"]
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    frames, act = torch.from_numpy(g["frames"]), torch.from_numpy(g["act"])
    with torch.no_grad():
        lr, le, hc = O.predict_rew_end(frames[:, 0:3], act[:, 0:3], frames[:, 1:4], sd, cfg)
        assert _rel(lr, torch.from_numpy(g["burn_rew"])) < 1e-4 and _rel(le, torch.from_numpy(g["burn_end"])) < 1e-4
        lr, le, hc = O.predict_rew_end(frames[:, 3:4], act[:, 3:4], frames[:, 4:5], sd, cfg, hc)
    assert _rel(lr, torch.from_numpy(g["step3_rew"])) < 1e-4 and _rel(le, torch.from_numpy(g["step3_end"])) < 1e-4
    assert _rel(hc[0], torch.from_numpy(g["hx"])) < 1e-5 and _rel(hc[1], torch.from_numpy(g["cx"])) < 1e-5


def _levels(cfg, channels):
    cfg.num_levels = len(channels)
    for i, ch in enumerate(channels):
        cfg.depths[i], cfg.channels[i], cfg.attn_depths[i] = 1, ch, 0


@pytest.mark.parametrize("channels", [[64, 256, 64], [256], [64, 96], [64, 128, 160]])
def test_create_refuses_levels_past_128(channels):
    lib = _lib.lib()
    bad = next(c for c in channels if c not in (32, 64, 128))
    d = _lib.DenoiserConfigC(img_channels=3, num_steps_conditioning=4, cond_channels=256, num_actions=4, sigma_data=0.5, sigma_offset_noise=0.3)
    _levels(d, channels)
    lib.dmd_launch_count(1)
    assert not lib.dmd_denoiser_create(d)
    err = lib.dmd_last_error().decode()
    assert "32, 64 or 128" in err and f"got {bad}" in err, err
    r = _lib.RewEndConfigC(lstm_dim=512, img_channels=3, img_size=64, cond_channels=128, num_actions=4)
    _levels(r, channels)
    assert not lib.dmd_rew_end_create(r)
    err = lib.dmd_last_error().decode()
    assert "32, 64 or 128" in err and f"got {bad}" in err, err
    assert lib.dmd_launch_count(0) == 0
