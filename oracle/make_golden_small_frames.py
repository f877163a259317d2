"""Generates the fixtures of frames smaller than 64 x 64 on the default 4-level nets, whose deepest level is then below 8 x 8, by
running the UNMODIFIED reference (oracle/ref_import.py) on seeded inputs and seeded 'de-zeroed' weights:

    DIAMOND_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_small_frames.py

- denoiser_32x32, denoiser_40x40, denoiser_32x64 (the schema of oracle/make_golden_frame_size.py): model output, denoised frame and
  a 3-step Euler trajectory.  The deepest levels are 4 x 4, 5 x 5 and 4 x 8; the mid-block attention runs over 16, 25 and 32 tokens.
- small_frames_training: Denoiser.forward + backward of the default net at 32 x 32 and 40 x 40 (SMALL_DENOISER_TRAIN, the layout
  of oracle/training_configs.DENOISER_CASES; draws replayed), and reward / termination training at 40 x 40 (SMALL_REW_END_TRAIN):
  losses and gradient summaries.
- actor_critic_small: the default actor-critic at img_size 40 and 84, where one level is odd (5 x 5, 21 x 21) and MaxPool2d floors
  it: predict_act_value over 3 recurrent steps, and the gradient of a fixed functional of the 3 steps' logits and values through
  the LSTM chain (BPTT), as a summary.

Weights and inputs are regenerated from the seeds below and guarded by stored checksums; the fixtures keep no weights.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import torch_oracle as O  # noqa: E402
from oracle import training_configs as TC  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

SMALL_FRAME_CASES = {
    "denoiser_32x32": dict(inner=O.InnerCfg(), h=32, w=32, b=2, wseed=3232, iseed=83, sigmas=[0.7, 3.0],
                           sampler=O.SamplerCfg(num_steps_denoising=3), rng_seed=10),
    "denoiser_40x40": dict(inner=O.InnerCfg(), h=40, w=40, b=2, wseed=4040, iseed=84, sigmas=[0.6, 2.5],
                           sampler=O.SamplerCfg(num_steps_denoising=3), rng_seed=11),
    "denoiser_32x64": dict(inner=O.InnerCfg(), h=32, w=64, b=2, wseed=3264, iseed=85, sigmas=[0.8, 4.0],
                           sampler=O.SamplerCfg(num_steps_denoising=3), rng_seed=12),
}

SMALL_DENOISER_TRAIN = {
    "S32": dict(inner=O.InnerCfg(), h=32, w=32, b=2, seq=1, mask_off=[], wseed=3240, dseed=3241),
    "S40": dict(inner=O.InnerCfg(), h=40, w=40, b=2, seq=2, mask_off=[(1, 5)], wseed=4050, dseed=4051),
}
SMALL_REW_END_TRAIN = {
    "R40": dict(cfg=O.RewEndCfg(img_size=40), b=4, T=7, death=(1, 3), pad=(2, 5), wseed=4060, dseed=4061),
}
SMALL_ACTOR_CRITIC = {
    "A40": dict(cfg=O.ActorCriticCfg(img_size=40), b=5, wseed=4070, dseed=4071),
    "A84": dict(cfg=O.ActorCriticCfg(img_size=84), b=3, wseed=8470, dseed=8471),
}
AC_STEPS = 3


def actor_critic_inputs(c):
    """obs [AC_STEPS, b, C, S, S] on the 1/255 grid, hx0 / cx0 [b, lstm_dim], and the weights (wl [AC_STEPS, b, A], wv
    [AC_STEPS, b]) of the functional sum_t <wl_t, logits_t> + <wv_t, val_t> whose gradient the fixture summarises."""
    cfg, b = c["cfg"], c["b"]
    rng = np.random.default_rng(c["dseed"])
    obs = torch.from_numpy(rng.integers(0, 256, size=(AC_STEPS, b, cfg.img_channels, cfg.img_size, cfg.img_size)).astype(np.float32))
    obs = obs.div(255).mul(2).sub(1)
    f = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32))  # noqa: E731
    return obs, f(b, cfg.lstm_dim) * 0.3, f(b, cfg.lstm_dim) * 0.3, f(AC_STEPS, b, cfg.num_actions), f(AC_STEPS, b)


def _summary(named):
    grads = [(k, p.grad) for k, p in named]
    assert all(g is not None for _, g in grads)
    return O.grad_summary(grads)


def make_denoiser_inference(ns):
    from oracle.make_golden import build_reference

    for name, c in SMALL_FRAME_CASES.items():
        inner, s = c["inner"], c["sampler"]
        assert s.order == 1 and s.s_churn == 0, "Euler without churn: the sampler draws nothing after x0"
        sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
        den = build_reference(ns, inner, sd)
        obs, act, x_noisy = O.synthetic_inputs(c["b"], inner, c["h"], c["w"], c["iseed"])
        sig = torch.tensor(c["sigmas"], dtype=torch.float32)
        b, t, ch, h, w = obs.shape
        with torch.no_grad():
            cs = den.compute_conditioners(sig)
            mo = den.compute_model_output(x_noisy, obs.reshape(b, t * ch, h, w), act, cs)
            dn = den.wrap_model_output(x_noisy, mo, cs)
            sampler = ns.diffusion.DiffusionSampler(den, ns.diffusion.DiffusionSamplerConfig(
                s.num_steps_denoising, s.sigma_min, s.sigma_max, s.rho, s.order, s.s_churn, s.s_tmin, s.s_tmax, s.s_noise))
            torch.manual_seed(c["rng_seed"])
            x, traj = sampler.sample(obs, act)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, weights_checksum=np.float64(O.state_checksum(sd)), sigmas_in=sig.numpy(), model_output=mo.numpy(),
                            denoised=dn.numpy(), sampler_sigmas=sampler.sigmas.numpy(), sample_x=x.numpy(), x0=traj[0].numpy(),
                            eps=np.zeros((len(sampler.sigmas) - 1, b, ch, h, w), np.float32), trajectory=torch.stack(traj).numpy())
        print(name, "model_output rms", float(mo.pow(2).mean().sqrt()), "size", os.path.getsize(path))


def _denoiser_training(ns, c):
    from oracle.make_golden import build_reference

    D = ns.diffusion
    sd = O.seeded_state_dict(O.inner_model_shapes(c["inner"]), c["wseed"])
    den = build_reference(ns, c["inner"], sd).train()
    sc = O.SigmaDistCfg()
    den.setup_training(D.SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    obs, act, mask, draws = TC.denoiser_inputs(c)
    b, T = obs.shape[:2]
    batch = ns.data.Batch(obs=obs.clone(), act=act, rew=torch.zeros(b, T), end=torch.zeros(b, T, dtype=torch.long),
                          trunc=torch.zeros(b, T, dtype=torch.long), mask_padding=mask, info=[{}] * b, segment_ids=[None] * b)
    q = [t for step in draws for t in step]
    randn, randn_like = torch.randn, torch.randn_like
    torch.randn = lambda *a, **k: q.pop(0).clone()
    torch.randn_like = lambda x, **k: q.pop(0).clone()
    try:
        loss, _ = den(batch)
    finally:
        torch.randn, torch.randn_like = randn, randn_like
    assert not q, "the reference consumed a different number of draws"
    loss.backward()
    keys, norms, samples = _summary(den.inner_model.named_parameters())
    return dict(weights_checksum=np.float64(O.state_checksum(sd)),
                inputs_checksum=np.float64(TC.inputs_checksum([obs, act, mask] + [t for s in draws for t in s])),
                loss=np.float64(loss.item()), grad_keys=np.array(keys), grad_norms=norms, grad_samples=samples)


def _rew_end_training(ns, c):
    cfg = c["cfg"]
    R = ns.rew_end_model
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"])
    m = R.RewEndModel(R.RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                          list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == O.rew_end_shapes(cfg)
    m.load_state_dict(sd)
    m.train()
    obs, act, rew, end, mask, final_obs = TC.rew_end_inputs(c)
    b = obs.size(0)
    info = [{"final_observation": final_obs[i]} if i in final_obs else {} for i in range(b)]
    batch = ns.data.Batch(obs=obs.clone(), act=act, rew=rew, end=end, trunc=torch.zeros_like(end), mask_padding=mask, info=info,
                          segment_ids=[None] * b)
    loss, _ = m(batch)
    loss.backward()
    keys, norms, samples = _summary(m.named_parameters())
    return dict(weights_checksum=np.float64(O.state_checksum(sd)),
                inputs_checksum=np.float64(TC.inputs_checksum([obs, act, rew, end, mask] + list(final_obs.values()))),
                loss=np.float64(loss.item()), grad_keys=np.array(keys), grad_norms=norms, grad_samples=samples)


def make_training(ns):
    out = {}
    for name, c in list(SMALL_DENOISER_TRAIN.items()) + list(SMALL_REW_END_TRAIN.items()):
        r = _denoiser_training(ns, c) if name in SMALL_DENOISER_TRAIN else _rew_end_training(ns, c)
        out.update({f"{name}_{k}": v for k, v in r.items()})
        print(name, "loss", float(r["loss"]))
    path = os.path.join(OUT, "small_frames_training.npz")
    np.savez_compressed(path, **out)
    print("training fixture size", os.path.getsize(path))


def make_actor_critic(ns):
    AC = ns.actor_critic
    out = {}
    for name, c in SMALL_ACTOR_CRITIC.items():
        cfg = c["cfg"]
        sd = O.seeded_actor_critic_state_dict(cfg, c["wseed"])
        ac = AC.ActorCritic(AC.ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down),
                                                 cfg.num_actions))
        assert [(k, tuple(v.shape)) for k, v in ac.state_dict().items()] == O.actor_critic_shapes(cfg)
        ac.load_state_dict(sd)
        obs, hx, cx, wl, wv = actor_critic_inputs(c)
        logits, vals = [], []
        h, cc = hx, cx
        for t in range(AC_STEPS):
            o = ac.predict_act_value(obs[t], (h, cc))
            logits.append(o.logits_act); vals.append(o.val); h, cc = o.hx_cx
        logits, vals = torch.stack(logits), torch.stack(vals)
        (logits * wl).sum().add((vals * wv).sum()).backward()
        keys, norms, samples = _summary(ac.named_parameters())
        out.update({f"{name}_weights_checksum": np.float64(O.state_checksum(sd)), f"{name}_logits": logits.detach().numpy(),
                    f"{name}_val": vals.detach().numpy(), f"{name}_hx": h.detach().numpy(), f"{name}_cx": cc.detach().numpy(),
                    f"{name}_grad_keys": np.array(keys), f"{name}_grad_norms": norms, f"{name}_grad_samples": samples})
        print(name, "logits rms", float(logits.detach().pow(2).mean().sqrt()))
    path = os.path.join(OUT, "actor_critic_small.npz")
    np.savez_compressed(path, **out)
    print("actor_critic_small size", os.path.getsize(path))


if __name__ == "__main__":
    from oracle import ref_import

    ns = ref_import.load()
    torch.set_num_threads(8)
    make_denoiser_inference(ns)
    make_training(ns)
    make_actor_critic(ns)
