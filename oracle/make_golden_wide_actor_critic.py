"""Generates tests/golden/actor_critic_wide.npz, the fixture of actor-critics with 128-channel levels, by running the
UNMODIFIED reference (imported as oracle/make_golden.py does) on seeded inputs and seeded 'de-zeroed' weights:

    DIAMOND_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_wide_actor_critic.py

Three policies (WIDE_AC_CASES): [64, 128, 128, 128] (3x3 128 -> 128 convs and a 64 -> 128 skip), [128] * 4 (a 128-channel conv0
and no skip), and [32, 128, 64, 128] (skip projections both ways across the 128 boundary).  Per case, keys prefixed "<name>/":
  - predict_act_value over FWD_STEPS recurrent steps at FWD_B rows from a random (hx, cx): logits, val, final hx / cx.  Rows
    are independent, so the first B rows are the reference at batch B;
  - ActorCritic.forward (the loss) through the reference's own make_env_loop over a scripted environment with a termination
    and a truncation (make_golden._ScriptedEnv), then backward: sampled actions, logits, values, loss, metrics and a gradient
    summary (torch_oracle.grad_summary), as actor_critic_training.npz.
Weights and frames are regenerated from their seeds (wide_ac_inputs) and guarded by a checksum and a digest.
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402
from oracle.make_golden import OUT, _ScriptedEnv  # noqa: E402

WIDE_AC_CASES = {
    "w64_128": dict(cfg=O.ActorCriticCfg(channels=[64, 128, 128, 128]), wseed=611, dseed=711),
    "w128": dict(cfg=O.ActorCriticCfg(channels=[128, 128, 128, 128]), wseed=612, dseed=712),
    "w32_128_64_128": dict(cfg=O.ActorCriticCfg(channels=[32, 128, 64, 128]), wseed=613, dseed=713),
}
FWD_B, FWD_STEPS = 32, 3
TRAIN_T, TRAIN_B = 5, 4
TRAIN_DEATHS = [(1, 2, "end"), (3, 0, "trunc")]   # (step, env, kind)
ACTION_SEED = 31


def _frames(u8) -> torch.Tensor:
    return torch.from_numpy(u8.astype(np.float32)).div(255).mul(2).sub(1)


def wide_ac_inputs(name) -> dict:
    """The inputs of one case, regenerated from its seed (numpy PCG64): forward frames [FWD_STEPS, FWD_B, C, H, W] with
    hx0 / cx0; the training rollout's obs_seq [T+1, b, C, H, W], rew / end / trunc [T, b] and final_obs {t: frames of the
    envs that died at t}; and `digest`, the SHA-256 of every frame."""
    c = WIDE_AC_CASES[name]
    cfg = c["cfg"]
    rng = np.random.default_rng(c["dseed"])
    img = (cfg.img_channels, cfg.img_size, cfg.img_size)
    fwd_u8 = rng.integers(0, 256, size=(FWD_STEPS, FWD_B) + img, dtype=np.uint8)
    hx0 = torch.from_numpy(rng.standard_normal((FWD_B, cfg.lstm_dim)).astype(np.float32)) * 0.3
    cx0 = torch.from_numpy(rng.standard_normal((FWD_B, cfg.lstm_dim)).astype(np.float32)) * 0.3
    obs_u8 = rng.integers(0, 256, size=(TRAIN_T + 1, TRAIN_B) + img, dtype=np.uint8)
    rew = torch.from_numpy(rng.choice([-1.0, 0.0, 0.0, 2.0], size=(TRAIN_T, TRAIN_B)).astype(np.float32))
    end = torch.zeros(TRAIN_T, TRAIN_B, dtype=torch.long)
    trunc = torch.zeros(TRAIN_T, TRAIN_B, dtype=torch.long)
    for t, e, kind in TRAIN_DEATHS:
        (end if kind == "end" else trunc)[t, e] = 1
    final_u8 = {t: rng.integers(0, 256, size=(1,) + img, dtype=np.uint8) for t, _, _ in TRAIN_DEATHS}
    h = hashlib.sha256(fwd_u8.tobytes())
    h.update(obs_u8.tobytes())
    for t in sorted(final_u8):
        h.update(final_u8[t].tobytes())
    return dict(fwd_obs=_frames(fwd_u8), hx0=hx0, cx0=cx0, obs_seq=_frames(obs_u8), rew=rew, end=end, trunc=trunc,
                final_obs={t: _frames(v) for t, v in final_u8.items()}, digest=h.hexdigest())


def make_case(ns, name) -> dict:
    c = WIDE_AC_CASES[name]
    cfg = c["cfg"]
    AC = ns.actor_critic
    sd = O.seeded_actor_critic_state_dict(cfg, c["wseed"])
    ac = AC.ActorCritic(AC.ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    assert [(k, tuple(v.shape)) for k, v in ac.state_dict().items()] == O.actor_critic_shapes(cfg)
    ac.load_state_dict(sd)
    x = wide_ac_inputs(name)
    out = {"weights_checksum": np.float64(O.state_checksum(sd)), "frames_sha256": np.array(x["digest"])}
    logits, vals = [], []
    hx, cx = x["hx0"], x["cx0"]
    with torch.no_grad():
        for t in range(FWD_STEPS):
            o = ac.predict_act_value(x["fwd_obs"][t], (hx, cx))
            logits.append(o.logits_act); vals.append(o.val); hx, cx = o.hx_cx
    out.update(fwd_logits=torch.stack(logits).numpy(), fwd_val=torch.stack(vals).numpy(), fwd_hx=hx.numpy(), fwd_cx=cx.numpy())

    lc = O.ActorCriticLossCfg(backup_every=TRAIN_T)
    env = _ScriptedEnv(x["obs_seq"], x["rew"], x["end"], x["trunc"], x["final_obs"], cfg.num_actions)
    ac.setup_training(env, AC.ActorCriticLossConfig(lc.backup_every, lc.gamma, lc.lambda_, lc.weight_value_loss, lc.weight_entropy_loss))
    torch.manual_seed(ACTION_SEED)
    captured = {}
    real_loop = ac.env_loop

    class _Tap:
        def send(self, n):
            captured["out"] = real_loop.send(n)
            return captured["out"]
    ac.env_loop = _Tap()
    loss, metrics = ac()
    loss.backward()
    _, act, _, _, _, lg, val, vb, _ = captured["out"]
    grads = [(k, p.grad) for k, p in ac.named_parameters()]
    assert all(g is not None for _, g in grads)
    keys, norms, samples = O.grad_summary(grads)
    out.update(act=act.numpy(), logits=lg.detach().numpy(), val=val.detach().numpy(), val_bootstrap=vb.numpy(),
               loss=np.float64(loss.item()), metric_keys=np.array(list(metrics.keys())),
               metric_vals=np.array([float(v) for v in metrics.values()], np.float64),
               grad_keys=np.array(keys), grad_norms=norms, grad_samples=samples)
    print(name, "logits rms", float(out["fwd_logits"].std()), "loss", loss.item(), "grad norm", float(np.sqrt((norms ** 2).sum())))
    return {f"{name}/{k}": v for k, v in out.items()}


if __name__ == "__main__":
    ns = ref_import.load()
    torch.set_num_threads(8)
    arrays = {}
    for name in WIDE_AC_CASES:
        arrays.update(make_case(ns, name))
    path = os.path.join(OUT, "actor_critic_wide.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, os.path.getsize(path), "bytes")
