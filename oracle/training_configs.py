"""Training cases beyond the two denoiser fixtures (tests/test_gpu_training_configs.py): the model configurations, their
seeded inputs, and the recipe that pins the oracle to the UNMODIFIED reference at two of them (D1, D4):

    DIAMOND_REFERENCE_SRC=<reference checkout>/src python oracle/training_configs.py

which writes tests/golden/training_config_{d1,d4}.npz (loss and gradient summary; the inputs are regenerated from the seeds
below and guarded by a checksum).  Frames are on the 1/255 grid in [-1, 1]; the standard-normal draws of the denoiser's
training step come from a torch.Generator, so the reference consumes them through a replayed torch.randn."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import torch_oracle as O  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

# denoiser cases: inner config, frame size, batch, autoregressive steps, (sample, frame) pairs masked off, seeds
DENOISER_CASES = {
    # a 64 -> 32 projection, a depth-3 level (4 up blocks), attention in the d / u blocks at C = 32 and a mid at C = 32
    "D1": dict(inner=O.InnerCfg(depths=[3, 1, 2, 1], channels=[64, 64, 32, 32], attn_depths=[0, 0, 0, 1]),
               h=64, w=64, b=2, seq=1, mask_off=[], wseed=601, dseed=611),
    # one level: no Down / Up records, the mid attention right after the d blocks
    "D2": dict(inner=O.InnerCfg(cond_channels=64, depths=[2], channels=[32], attn_depths=[0]),
               h=8, w=8, b=3, seq=1, mask_off=[], wseed=602, dseed=612),
    # non-square frames at every level, 64-token attention laid out as 4 x 16
    "D3": dict(inner=O.InnerCfg(), h=32, w=128, b=2, seq=1, mask_off=[], wseed=603, dseed=613),
    # 12 output channels (the output gradient past 8 channels), a three-pass split-fp16 conv_in (60 -> 64 channels) in a
    # training forward, projections 64 -> 32 and 32 -> 64
    "D4": dict(inner=O.InnerCfg(img_channels=12, num_steps_conditioning=4, cond_channels=128, depths=[1, 1, 1],
                                channels=[64, 32, 64], attn_depths=[0, 0, 0], num_actions=18),
               h=32, w=32, b=2, seq=1, mask_off=[], wseed=604, dseed=614),
    # the smallest FiLM table and split-K (cond 32), a batch of one
    "D5": dict(inner=O.InnerCfg(img_channels=1, num_steps_conditioning=1, cond_channels=32, depths=[1, 1, 1],
                                channels=[32, 32, 32], attn_depths=[0, 0, 0], num_actions=2),
               h=32, w=32, b=1, seq=1, mask_off=[], wseed=605, dseed=615),
    # the small-net fixture's config over 3 autoregressive steps: sample 0 padded on every predicted step, sample 1 on the
    # middle one
    "D6": dict(inner=O.InnerCfg(img_channels=3, num_steps_conditioning=2, cond_channels=64, depths=[1, 2, 1],
                                channels=[32, 64, 32], attn_depths=[0, 0, 1], num_actions=6),
               h=32, w=32, b=3, seq=3, mask_off=[(0, 2), (0, 3), (0, 4), (1, 3)], wseed=606, dseed=616),
}

# reward / termination cases: config, segments x frames, the segment that dies (at step t, with a final observation) and
# the one whose tail is padding (from step t on)
REW_END_CASES = {
    "R1": dict(cfg=O.RewEndCfg(cond_channels=64, channels=[32, 32, 64, 64], attn_depths=[0, 0, 0, 1]),
               b=4, T=7, death=(1, 3), pad=(2, 5), wseed=621, dseed=631),
    "R2": dict(cfg=O.RewEndCfg(lstm_dim=256, img_channels=1, img_size=32, cond_channels=256, depths=[1, 3, 1],
                               channels=[64, 64, 32], attn_depths=[0, 0, 1], num_actions=18),
               b=5, T=4, death=(3, 1), pad=(0, 2), wseed=622, dseed=632),
}

# actor-critic cases: config, envs x steps, one termination (step, env) and one truncation (step, env)
ACTOR_CRITIC_CASES = {
    "A1": dict(cfg=O.ActorCriticCfg(lstm_dim=256, img_channels=3, img_size=64, channels=[32, 64, 32, 64], down=[1, 0, 1, 1],
                                    num_actions=18), b=4, T=6, end=(2, 1), trunc=(4, 3), wseed=641, dseed=651),
    "A2": dict(cfg=O.ActorCriticCfg(lstm_dim=128, img_channels=1, img_size=32, channels=[64, 64], down=[0, 1], num_actions=4),
               b=3, T=5, end=(1, 0), trunc=(3, 2), wseed=642, dseed=652),
}

# the cases pinned to the reference by tests/golden/training_config_<id>.npz
GOLDEN_CASES = ("D1", "D4")


def _frames(rng, shape):
    return torch.from_numpy(rng.integers(0, 256, size=shape).astype(np.float32)).div(255).mul(2).sub(1)


def denoiser_inputs(c):
    """(obs [b, n + seq, c, h, w], act [b, n + seq], mask_padding [b, n + seq], draws: per step (raw_sigma [b],
    raw_offset [b, c, 1, 1], raw_noise [b, c, h, w])), float32."""
    inner, b, h, w = c["inner"], c["b"], c["h"], c["w"]
    T = inner.num_steps_conditioning + c["seq"]
    rng = np.random.default_rng(c["dseed"])
    obs = _frames(rng, (b, T, inner.img_channels, h, w))
    act = torch.from_numpy(rng.integers(0, inner.num_actions, size=(b, T)).astype(np.int64))
    mask = torch.ones(b, T, dtype=torch.bool)
    for bi, ti in c["mask_off"]:
        mask[bi, ti] = False
    g = torch.Generator().manual_seed(c["dseed"])
    draws = [(torch.randn(b, generator=g), torch.randn(b, inner.img_channels, 1, 1, generator=g),
              torch.randn(b, inner.img_channels, h, w, generator=g)) for _ in range(c["seq"])]
    return obs, act, mask, draws


def rew_end_inputs(c):
    """(obs [b, T, c, h, w], act, rew, end, mask_padding [b, T], final_obs {segment: frame}) as rew_end_training.golden_inputs:
    one segment dies at its `death` step and carries a final observation, one runs into padding; rewards of every sign."""
    cfg, b, T = c["cfg"], c["b"], c["T"]
    rng = np.random.default_rng(c["dseed"])
    obs = _frames(rng, (b, T, cfg.img_channels, cfg.img_size, cfg.img_size))
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, T)).astype(np.int64))
    rew = torch.from_numpy(rng.choice([-3.0, -1.0, 0.0, 0.0, 0.5, 1.0, 2.5], size=(b, T)).astype(np.float32))
    end = torch.zeros(b, T, dtype=torch.long)
    mask = torch.ones(b, T, dtype=torch.bool)
    (di, dt), (pi, pt) = c["death"], c["pad"]
    end[di, dt] = 1
    for i, t0 in ((di, dt + 1), (pi, pt)):   # padding: uint8 127, on the 1/255 grid
        mask[i, t0:] = False
        obs[i, t0:] = 127 / 255 * 2 - 1
        rew[i, t0:] = 0
        act[i, t0:] = 0
    final_obs = {di: _frames(rng, (cfg.img_channels, cfg.img_size, cfg.img_size))}
    return obs, act, rew, end, mask, final_obs


def actor_critic_inputs(c):
    """A scripted environment's rollout: obs_seq [T + 1, b, c, h, w], rew / end / trunc [T, b], final_obs {t: [k, c, h, w]}
    for the envs that die at step t, and the actions the policy is made to take, act [b, T]."""
    cfg, b, T = c["cfg"], c["b"], c["T"]
    rng = np.random.default_rng(c["dseed"])
    obs_seq = _frames(rng, (T + 1, b, cfg.img_channels, cfg.img_size, cfg.img_size))
    rew = torch.from_numpy(rng.choice([-2.0, -1.0, 0.0, 0.0, 1.0, 3.0], size=(T, b)).astype(np.float32))
    end = torch.zeros(T, b, dtype=torch.long)
    trunc = torch.zeros(T, b, dtype=torch.long)
    end[c["end"]] = 1
    trunc[c["trunc"]] = 1
    final_obs = {t: _frames(rng, (1, cfg.img_channels, cfg.img_size, cfg.img_size)) for t in (c["end"][0], c["trunc"][0])}
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, T)).astype(np.int64))
    return obs_seq, rew, end, trunc, final_obs, act


def inputs_checksum(tensors) -> float:
    return float(sum(t.double().abs().sum() for t in tensors))


def make_goldens():
    """The reference's Denoiser.forward + backward at GOLDEN_CASES, its draws replayed from denoiser_inputs."""
    from oracle import ref_import
    from oracle.make_golden import build_reference

    ns = ref_import.load()
    D = ns.diffusion
    torch.set_num_threads(8)
    for name in GOLDEN_CASES:
        c = DENOISER_CASES[name]
        inner = c["inner"]
        sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
        den = build_reference(ns, inner, sd).train()
        sc = O.SigmaDistCfg()
        den.setup_training(D.SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
        obs, act, mask, draws = denoiser_inputs(c)
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
        grads = [(k, p.grad) for k, p in den.inner_model.named_parameters()]
        assert all(g is not None for _, g in grads)
        keys, norms, samples = O.grad_summary(grads)
        path = os.path.join(GOLDEN_DIR, f"training_config_{name.lower()}.npz")
        np.savez_compressed(path, weights_checksum=np.float64(O.state_checksum(sd)),
                            inputs_checksum=np.float64(inputs_checksum([obs, act, mask] + [t for s in draws for t in s])),
                            loss=np.float64(loss.item()), grad_keys=np.array(keys), grad_norms=norms, grad_samples=samples)
        print(name, "loss", loss.item(), "grad norm", float(np.sqrt((norms ** 2).sum())), "size", os.path.getsize(path))


if __name__ == "__main__":
    make_goldens()
