"""CPU: actor-critics with 128-channel levels.  The float32 oracle (oracle/torch_oracle.py) reproduces the reference's own
forward outputs, loss and gradients for the three policies of tests/golden/actor_critic_wide.npz (written by
oracle/make_golden_wide_actor_critic.py), and dmd_actor_critic_create takes 32, 64 or 128 channels per level in any mix and
refuses any other width, naming the limit and the level, before it touches a device."""
import itertools
import os

import numpy as np
import pytest
import torch

from diamond_b200 import _lib
from oracle import torch_oracle as O
from oracle.make_golden_wide_actor_critic import FWD_STEPS, TRAIN_T, WIDE_AC_CASES, wide_ac_inputs


def _rel(a, b):
    return float((a - b).double().norm() / b.double().norm().clamp_min(1e-300))


def _golden(golden_dir, name):
    g = np.load(os.path.join(golden_dir, "actor_critic_wide.npz"))
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


def _check_grads(named_grads, g, rtol_norm=2e-4):
    """The tolerance of the actor-critic training fixture (tests/test_oracle_training_golden.py)."""
    keys, norms, samples = O.grad_summary(named_grads)
    assert keys == [str(k) for k in g["grad_keys"]]
    ref_n, ref_s = g["grad_norms"], g["grad_samples"]
    total = float(np.sqrt((ref_n ** 2).sum()))
    assert np.all(np.abs(norms - ref_n) <= rtol_norm * ref_n + 1e-6 * total), float(np.max(np.abs(norms - ref_n) / (ref_n + 1e-12)))
    numel = np.array([gr.numel() for _, gr in named_grads], np.float64)
    scale = (ref_n / np.sqrt(numel))[:, None]
    assert np.all(np.abs(samples - ref_s) <= 2e-4 * np.abs(ref_s) + 2e-3 * scale + 1e-9)


@pytest.mark.parametrize("name", list(WIDE_AC_CASES))
def test_oracle_matches_wide_actor_critic_golden(golden_dir, name):
    torch.set_num_threads(8)
    c = WIDE_AC_CASES[name]
    cfg = c["cfg"]
    g = _golden(golden_dir, name)
    sd = O.seeded_actor_critic_state_dict(cfg, c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    x = wide_ac_inputs(name)
    assert x["digest"] == str(g["frames_sha256"]), "regenerated frames differ from the fixture's"
    hx, cx = x["hx0"], x["cx0"]
    with torch.no_grad():
        for t in range(FWD_STEPS):
            logits, val, (hx, cx) = O.predict_act_value(x["fwd_obs"][t], hx, cx, sd, cfg)
            assert _rel(logits, torch.from_numpy(g["fwd_logits"][t])) < 1e-5
            assert _rel(val, torch.from_numpy(g["fwd_val"][t])) < 1e-5
    assert _rel(hx, torch.from_numpy(g["fwd_hx"])) < 1e-5 and _rel(cx, torch.from_numpy(g["fwd_cx"])) < 1e-5

    for v in sd.values():
        v.requires_grad_(True)
    logits, val, vb = O.actor_critic_rollout(x["obs_seq"], x["end"], x["trunc"], x["final_obs"], sd, cfg)
    assert torch.allclose(logits, torch.from_numpy(g["logits"]), rtol=1e-4, atol=1e-5)
    assert torch.allclose(val, torch.from_numpy(g["val"]), rtol=1e-4, atol=1e-5)
    assert torch.allclose(vb, torch.from_numpy(g["val_bootstrap"]), rtol=1e-4, atol=1e-5)
    lc = O.ActorCriticLossCfg(backup_every=TRAIN_T)
    loss, metrics = O.actor_critic_loss(logits, val, torch.from_numpy(g["act"]), x["rew"].t(), x["end"].t(), x["trunc"].t(), vb, lc)
    assert abs(loss.item() - float(g["loss"])) <= 2e-5 * abs(float(g["loss"])), (loss.item(), float(g["loss"]))
    for k, v in zip(g["metric_keys"], g["metric_vals"]):
        assert abs(float(metrics[str(k)]) - float(v)) <= 1e-4 * abs(float(v)) + 1e-7, k
    loss.backward()
    _check_grads([(k, v.grad) for k, v in sd.items()], g)


def _config(channels):
    c = _lib.ActorCriticConfigC(lstm_dim=512, img_channels=3, img_size=64, num_levels=len(channels), num_actions=4)
    for i, ch in enumerate(channels):
        c.channels[i], c.down[i] = ch, 1
    return c


@pytest.mark.parametrize("channels", [[96], [64, 96, 64, 64], [32, 64, 128, 160], [128, 256], [256, 128, 128, 128]])
def test_create_refuses_other_widths(channels):
    lib = _lib.lib()
    bad_level, bad = next((i, c) for i, c in enumerate(channels) if c not in (32, 64, 128))
    lib.dmd_launch_count(1)
    assert not lib.dmd_actor_critic_create(_config(channels))
    err = lib.dmd_last_error().decode()
    assert "32, 64 or 128" in err and f"got {bad} at level {bad_level}" in err, err
    assert lib.dmd_launch_count(0) == 0


def test_create_width_check_accepts_every_mix():
    """Every mix of 32, 64 and 128 over four levels passes the width validation: create does not fail with its message.
    This is all a host without a device can check, since create queries the device next;
    tests/test_gpu_actor_critic_wide.py creates every mix on the GPU."""
    lib = _lib.lib()
    for channels in itertools.product([32, 64, 128], repeat=4):
        h = lib.dmd_actor_critic_create(_config(list(channels)))
        if h:
            lib.dmd_actor_critic_destroy(h)
            continue
        err = lib.dmd_last_error().decode()
        assert "channels must" not in err, (channels, err)
