"""CPU: conditioning vectors wider than 256 channels.  The float32 oracle (oracle/torch_oracle.py) reproduces the reference's
own outputs and training gradients for a cond_channels = 2048 denoiser and a cond_channels = 512 reward / termination model
(tests/golden/denoiser_cond2048.npz, rew_end_cond512.npz, written by oracle/make_golden_cond.py), and the executors' create
calls accept every multiple of 32 up to 2048 and refuse anything else, naming the limit, before they touch a device."""
import os

import numpy as np
import pytest
import torch

from diamond_b200 import _lib


def _rel(a, b):
    return float((a - b).double().norm() / b.double().norm().clamp_min(1e-300))


def _check_summary(g, named, rtol=2e-4):
    """named [(key, grad)] against the fixture's gradient summary (training_config goldens' tolerances)."""
    from oracle import torch_oracle as O

    keys, norms, samples = O.grad_summary(named)
    assert keys == [str(k) for k in g["grad_keys"]]
    ref_n, ref_s = g["grad_norms"], g["grad_samples"]
    total = float(np.sqrt((ref_n ** 2).sum()))
    assert np.all(np.abs(norms - ref_n) <= rtol * ref_n + 1e-6 * total), float(np.max(np.abs(norms - ref_n) / (ref_n + 1e-12)))
    numel = np.array([gr.numel() for _, gr in named], np.float64)
    scale = (ref_n / np.sqrt(numel))[:, None]
    assert np.all(np.abs(samples - ref_s) <= rtol * np.abs(ref_s) + 2e-3 * scale + 1e-9)


def test_oracle_matches_cond2048_denoiser_golden(golden_dir):
    from oracle import torch_oracle as O
    from oracle.make_golden_cond import DENOISER_COND as c

    g = np.load(os.path.join(golden_dir, "denoiser_cond2048.npz"))
    inner = c["inner"]
    assert inner.cond_channels == 2048
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    obs, act, x_noisy = O.synthetic_inputs(c["b"], inner, c["h"], c["w"], c["iseed"])
    b, t, ch, h, w = obs.shape
    cfg = O.DenoiserCfg(inner=inner)
    with torch.no_grad():
        mo = O.model_output(x_noisy, torch.from_numpy(g["sigmas_in"]), obs.reshape(b, t * ch, h, w), act, sd, cfg)
        x, traj = O.sample(obs, act, torch.from_numpy(g["x0"]), sd, cfg, c["sampler"])
    assert _rel(mo, torch.from_numpy(g["model_output"])) < 1e-5
    # the sampler quantises every denoised frame (denoiser.py:83): a pixel on a bucket edge may round the other way
    assert float((x - torch.from_numpy(g["sample_x"])).abs().gt(1e-3).float().mean()) < 0.02


def test_oracle_training_matches_cond2048_denoiser_golden(golden_dir):
    from oracle import torch_oracle as O
    from oracle import training_configs as TC
    from oracle.make_golden_cond import denoiser_train_case

    g = np.load(os.path.join(golden_dir, "denoiser_cond2048.npz"))
    c = denoiser_train_case()
    obs, act, mask, draws = TC.denoiser_inputs(c)
    assert abs(TC.inputs_checksum([obs, act, mask] + [t for s in draws for t in s]) - float(g["train_inputs_checksum"])) \
        < 1e-9 * float(g["train_inputs_checksum"])
    sd = O.seeded_state_dict(O.inner_model_shapes(c["inner"]), c["wseed"])
    for k, v in sd.items():
        v.requires_grad_(k != "noise_emb.weight")
    loss = O.denoiser_loss(obs, act, mask, draws, sd, O.DenoiserCfg(inner=c["inner"]), O.SigmaDistCfg())
    assert abs(loss.item() - float(g["train_loss"])) <= 2e-5 * abs(float(g["train_loss"]))
    loss.backward()
    _check_summary(g, [(k, v.grad) for k, v in sd.items() if k != "noise_emb.weight"])


def test_oracle_matches_cond512_rew_end_golden(golden_dir):
    from oracle import rew_end_training as RT
    from oracle import torch_oracle as O
    from oracle import training_configs as TC
    from oracle.make_golden_cond import REW_END_COND as c
    from oracle.make_golden_cond import rew_end_predict_inputs, rew_end_train_case

    g = np.load(os.path.join(golden_dir, "rew_end_cond512.npz"))
    cfg = c["cfg"]
    assert cfg.cond_channels == 512
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    frames, act = rew_end_predict_inputs()
    assert torch.equal(frames, torch.from_numpy(g["frames"])) and torch.equal(act, torch.from_numpy(g["act"]))
    with torch.no_grad():
        lr, le, hc = O.predict_rew_end(frames[:, 0:3], act[:, 0:3], frames[:, 1:4], sd, cfg)
        assert _rel(lr, torch.from_numpy(g["burn_rew"])) < 1e-4 and _rel(le, torch.from_numpy(g["burn_end"])) < 1e-4
        lr, le, hc = O.predict_rew_end(frames[:, 3:4], act[:, 3:4], frames[:, 4:5], sd, cfg, hc)
    assert _rel(lr, torch.from_numpy(g["step3_rew"])) < 1e-4 and _rel(le, torch.from_numpy(g["step3_end"])) < 1e-4
    assert _rel(hc[0], torch.from_numpy(g["hx"])) < 1e-5 and _rel(hc[1], torch.from_numpy(g["cx"])) < 1e-5

    obs, tact, rew, end, mask, final_obs = TC.rew_end_inputs(rew_end_train_case())
    assert abs(TC.inputs_checksum([obs, tact, rew, end, mask] + list(final_obs.values())) - float(g["train_inputs_checksum"])) \
        < 1e-9 * float(g["train_inputs_checksum"])
    for v in sd.values():
        v.requires_grad_(True)
    loss = RT.rew_end_loss(obs, tact, rew, end, mask, final_obs, sd, cfg)[0]
    assert abs(loss.item() - float(g["train_loss"])) <= 2e-5 * abs(float(g["train_loss"]))
    loss.backward()
    _check_summary(g, [(k, v.grad) for k, v in sd.items()])


def _configs(cc):
    d = _lib.DenoiserConfigC(img_channels=3, num_steps_conditioning=4, cond_channels=cc, num_actions=4, sigma_data=0.5,
                             sigma_offset_noise=0.3)
    r = _lib.RewEndConfigC(lstm_dim=512, img_channels=3, img_size=64, cond_channels=cc, num_actions=4)
    for cfg in (d, r):
        cfg.num_levels = 2
        for i, ch in enumerate((64, 128)):
            cfg.depths[i], cfg.channels[i], cfg.attn_depths[i] = 1, ch, 0
    return d, r


@pytest.mark.parametrize("cc", [2080, 4096, 48, 100])
def test_create_refuses_cond_channels_past_2048_or_off_32(cc):
    lib = _lib.lib()
    d, r = _configs(cc)
    lib.dmd_launch_count(1)
    assert not lib.dmd_denoiser_create(d)
    err = lib.dmd_last_error().decode()
    assert "cond_channels" in err and "2048" in err and f"got {cc}" in err, err
    assert not lib.dmd_rew_end_create(r)
    err = lib.dmd_last_error().decode()
    assert "cond_channels" in err and "2048" in err and f"got {cc}" in err, err
    assert lib.dmd_launch_count(0) == 0


def test_create_refuses_cond_channels_off_the_frame_stack():
    lib = _lib.lib()
    d, _ = _configs(288)
    d.num_steps_conditioning = 5   # 288 = 32 x 9 is not a multiple of 5
    assert not lib.dmd_denoiser_create(d)
    err = lib.dmd_last_error().decode()
    assert "num_steps_conditioning" in err and "got 288" in err, err


@pytest.mark.parametrize("cc", [288, 512, 1024, 2048])
def test_create_accepts_cond_channels_up_to_2048_before_any_device_work(cc):
    """Past the cond_channels check, create fails only at its first device allocation on a machine without a GPU; the error
    it gives is then not about cond_channels."""
    lib = _lib.lib()
    d, r = _configs(cc)
    lib.dmd_launch_count(1)
    for create, destroy, cfg in ((lib.dmd_denoiser_create, lib.dmd_denoiser_destroy, d),
                                 (lib.dmd_rew_end_create, lib.dmd_rew_end_destroy, r)):
        h = create(cfg)
        if h:
            destroy(h)
        else:
            err = lib.dmd_last_error().decode()
            assert "cond_channels" not in err and "channels must be" not in err, err
    assert lib.dmd_launch_count(0) == 0
