"""CPU: frames smaller than 64 x 64.  The float32 oracle (oracle/torch_oracle.py) reproduces the reference's own outputs at
32 x 32, 40 x 40 and 32 x 64, its training losses and gradients at 32 and 40, and the actor-critic's forward and BPTT gradient
at img_size 40 and 84 (tests/golden/denoiser_{32x32,40x40,32x64}.npz, small_frames_training.npz, actor_critic_small.npz,
written by oracle/make_golden_small_frames.py).  The executors' create calls and host-side planners accept these sizes."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from diamond_b200 import _lib
from oracle import make_golden_small_frames as SF
from oracle import rew_end_training as RT
from oracle import torch_oracle as O
from oracle import training_configs as TC

HERE = os.path.dirname(os.path.abspath(__file__))
P = 0x1000  # any non-null address


def _load(name):
    spec = importlib.util.spec_from_file_location(f"_small_frames_{name}", os.path.join(HERE, name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


CW = _load("test_cond_width_host")


@pytest.mark.parametrize("name", list(SF.SMALL_FRAME_CASES))
def test_oracle_matches_reference_golden_at_small_frames(golden_dir, name):
    c = SF.SMALL_FRAME_CASES[name]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
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
    s = c["sampler"]
    assert torch.equal(O.build_sigmas(s.num_steps_denoising, s.sigma_min, s.sigma_max, s.rho), torch.from_numpy(g["sampler_sigmas"]))
    x0 = torch.from_numpy(g["x0"])
    with torch.no_grad():
        x, traj = O.sample(obs, act, x0, sd, cfg, s)
    diff = (torch.stack(traj) - torch.from_numpy(g["trajectory"])).abs()
    assert float((diff > 1e-4).float().mean()) < 2e-3, float(diff.max())


def _fixture(golden_dir, name, prefix):
    g = np.load(os.path.join(golden_dir, name))
    return {k[len(prefix) + 1:]: g[k] for k in g.files if k.startswith(prefix + "_")}


@pytest.mark.parametrize("name", list(SF.SMALL_DENOISER_TRAIN) + list(SF.SMALL_REW_END_TRAIN))
def test_oracle_training_matches_reference_golden_at_small_frames(golden_dir, name):
    g = _fixture(golden_dir, "small_frames_training.npz", name)
    torch.set_num_threads(8)
    if name in SF.SMALL_DENOISER_TRAIN:
        c = SF.SMALL_DENOISER_TRAIN[name]
        sd = O.seeded_state_dict(O.inner_model_shapes(c["inner"]), c["wseed"])
        obs, act, mask, draws = TC.denoiser_inputs(c)
        assert abs(TC.inputs_checksum([obs, act, mask] + [t for s in draws for t in s]) - float(g["inputs_checksum"])) < 1e-9 * float(g["inputs_checksum"])
        for k, v in sd.items():
            if k != "noise_emb.weight":
                v.requires_grad_(True)
        loss = O.denoiser_loss(obs, act, mask, draws, sd, O.DenoiserCfg(inner=c["inner"]), O.SigmaDistCfg())
        loss.backward()
        named = [(k, v.grad) for k, v in sd.items() if k != "noise_emb.weight"]
    else:
        c = SF.SMALL_REW_END_TRAIN[name]
        sd = O.seeded_state_dict(O.rew_end_shapes(c["cfg"]), c["wseed"])
        obs, act, rew, end, mask, final_obs = TC.rew_end_inputs(c)
        for v in sd.values():
            v.requires_grad_(True)
        loss = RT.rew_end_loss(obs, act, rew, end, mask, final_obs, sd, c["cfg"])[0]
        loss.backward()
        named = [(k, v.grad) for k, v in sd.items()]
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * abs(float(g["weights_checksum"]))
    assert abs(loss.item() - float(g["loss"])) <= 2e-5 * abs(float(g["loss"])), (loss.item(), float(g["loss"]))
    CW._check_summary(g, named)


@pytest.mark.parametrize("name", list(SF.SMALL_ACTOR_CRITIC))
def test_oracle_actor_critic_matches_reference_golden_at_odd_levels(golden_dir, name):
    """Forward over 3 recurrent steps and the BPTT gradient; at img_size 40 the last level pools 5 x 5 to 2 x 2, at 84 the third
    pools 21 x 21 to 10 x 10 (floor division, as nn.MaxPool2d)."""
    c = SF.SMALL_ACTOR_CRITIC[name]
    cfg = c["cfg"]
    g = _fixture(golden_dir, "actor_critic_small.npz", name)
    sd = O.seeded_actor_critic_state_dict(cfg, c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * abs(float(g["weights_checksum"]))
    for v in sd.values():
        v.requires_grad_(True)
    obs, h, cx, wl, wv = SF.actor_critic_inputs(c)
    logits, vals = [], []
    for t in range(SF.AC_STEPS):
        lg, val, (h, cx) = O.predict_act_value(obs[t], h, cx, sd, cfg)
        logits.append(lg); vals.append(val)
    logits, vals = torch.stack(logits), torch.stack(vals)
    for k, v in (("logits", logits), ("val", vals), ("hx", h), ("cx", cx)):
        assert torch.allclose(v.detach(), torch.from_numpy(g[k]), rtol=1e-5, atol=1e-5), (k, float((v.detach() - torch.from_numpy(g[k])).abs().max()))
    (logits * wl).sum().add((vals * wv).sum()).backward()
    CW._check_summary(g, [(k, v.grad) for k, v in sd.items()])


def test_small_frame_fixtures_fit_their_budget(golden_dir):
    names = [n + ".npz" for n in SF.SMALL_FRAME_CASES] + ["small_frames_training.npz", "actor_critic_small.npz"]
    sizes = [os.path.getsize(os.path.join(golden_dir, n)) for n in names]
    assert max(sizes) < 1_000_000 and sum(sizes) <= 1024 * 1024, sizes


# ------------------------------------------------------------------------------------------------ host-side planning
def _prep(**kw):
    lib = _lib.lib()
    d = _lib.PrepDesc()
    for k, v in dict(dict(src0=P, dst0=P, C0=64, B=32, Hs=4, Ws=4), **kw).items():
        setattr(d, k, v)
    blocks, ppb, nsrc = C.c_int(), C.c_int(), C.c_int()
    rc = lib.dmd_prep_plan(C.byref(d), C.byref(blocks), C.byref(ppb), C.byref(nsrc))
    return rc, blocks.value, ppb.value, lib.dmd_last_error().decode()


@pytest.mark.parametrize("hw", [(4, 4), (4, 8), (5, 5), (6, 6), (7, 7)])
def test_prep_plans_levels_down_to_4x4(hw):
    """A prep block touches at most two images: on a 4 x 4 image (25 padded positions) it takes 16 positions."""
    rc, blocks, ppb, err = _prep(Hs=hw[0], Ws=hw[1])
    assert rc == 0, err
    assert ppb <= (hw[0] + 1) * (hw[1] + 1) and ppb % 16 == 0
    if hw == (4, 4):
        assert ppb == 16


@pytest.mark.parametrize("hw", [(2, 2), (3, 3), (2, 6)])
def test_prep_refuses_levels_below_4x4(hw):
    rc, _, _, err = _prep(Hs=hw[0], Ws=hw[1])
    assert rc != 0 and "image too small" in err, err


def _denoiser_config(levels=4):
    d = _lib.DenoiserConfigC(img_channels=3, num_steps_conditioning=4, cond_channels=256, num_actions=4, sigma_data=0.5,
                             sigma_offset_noise=0.3)
    d.num_levels = levels
    for i in range(levels):
        d.depths[i], d.channels[i], d.attn_depths[i] = 2, 64, 0
    return d


@pytest.mark.parametrize("levels", [4, 5])
def test_create_accepts_the_default_nets_and_five_levels_before_any_device_work(levels):
    """Past its config checks, create fails only at its first device allocation on a machine without a GPU; the frame size
    is chosen per call, so nothing at create time depends on it."""
    lib = _lib.lib()
    lib.dmd_launch_count(1)
    h = lib.dmd_denoiser_create(_denoiser_config(levels))
    if h:
        lib.dmd_denoiser_destroy(h)
    else:
        err = lib.dmd_last_error().decode()
        assert "channels must be" not in err and "levels" not in err, err
    assert lib.dmd_launch_count(0) == 0
