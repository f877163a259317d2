"""Generates the fixtures of nets with 128-channel levels (tests/golden/denoiser_wide.npz, rew_end_wide.npz) by running the
UNMODIFIED reference (imported as oracle/make_golden.py does) on seeded inputs and seeded 'de-zeroed' weights:

    DIAMOND_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_wide.py

denoiser_wide: a [64, 128, 128, 128] U-Net (its 128 -> 128 convs, 256-channel up-path concats and 256 -> 128 skip projections
run K-split, its mid-block attention at C = 128): model output, denoised frame and an Euler sampler trajectory.
rew_end_wide: a [128] * 4 reward / termination encoder (attention at C = 128 in its last two ResBlocks): a 3-step burn-in
call, then one step carrying the LSTM state.  Weights are regenerated from the seed and guarded by a stored checksum.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402
from oracle.make_golden import OUT, build_reference  # noqa: E402

DENOISER_WIDE = dict(
    inner=O.InnerCfg(depths=[1, 1, 1, 1], channels=[64, 128, 128, 128]), h=64, w=64, b=2, wseed=2468, iseed=80,
    sigmas=[0.7, 3.0], sampler=O.SamplerCfg(num_steps_denoising=3), rng_seed=7,
)
REW_END_WIDE = dict(cfg=O.RewEndCfg(depths=[1, 1, 1, 1], channels=[128, 128, 128, 128]), wseed=779, dseed=94, b=2)


def make_denoiser_wide(ns):
    c = DENOISER_WIDE
    inner = c["inner"]
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    den = build_reference(ns, inner, sd)
    obs, act, x_noisy = O.synthetic_inputs(c["b"], inner, c["h"], c["w"], c["iseed"])
    sig = torch.tensor(c["sigmas"], dtype=torch.float32)
    b, t, ch, h, w = obs.shape
    obs_flat = obs.reshape(b, t * ch, h, w)
    s = c["sampler"]
    assert s.order == 1 and s.s_churn == 0   # the sampler draws only x0
    with torch.no_grad():
        cs = den.compute_conditioners(sig)
        mo = den.compute_model_output(x_noisy, obs_flat, act, cs)
        dn = den.wrap_model_output(x_noisy, mo, cs)
        sampler = ns.diffusion.DiffusionSampler(den, ns.diffusion.DiffusionSamplerConfig(
            s.num_steps_denoising, s.sigma_min, s.sigma_max, s.rho, s.order, s.s_churn, s.s_tmin, s.s_tmax, s.s_noise))
        torch.manual_seed(c["rng_seed"])
        x, traj = sampler.sample(obs, act)
    path = os.path.join(OUT, "denoiser_wide.npz")
    np.savez_compressed(path, weights_checksum=np.float64(O.state_checksum(sd)), sigmas_in=sig.numpy(), model_output=mo.numpy(),
                        denoised=dn.numpy(), sampler_sigmas=sampler.sigmas.numpy(), x0=traj[0].numpy(), sample_x=x.numpy(),
                        trajectory=torch.stack(traj).numpy())
    print("denoiser_wide model_output rms", float(mo.pow(2).mean().sqrt()), "size", os.path.getsize(path))


def make_rew_end_wide(ns):
    c = REW_END_WIDE
    cfg, b = c["cfg"], c["b"]
    R = ns.rew_end_model
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"])
    m = R.RewEndModel(R.RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                          list(cfg.channels), list(cfg.attn_depths), cfg.num_actions)).eval()
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == O.rew_end_shapes(cfg)
    m.load_state_dict(sd)
    rng = np.random.default_rng(c["dseed"])
    frames = torch.from_numpy(rng.integers(0, 256, size=(b, 5, 3, 64, 64)).astype(np.float32)).div(255).mul(2).sub(1)
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, 4)).astype(np.int64))
    with torch.no_grad():
        br, be, hc = m.predict_rew_end(frames[:, 0:3], act[:, 0:3], frames[:, 1:4])
        sr, se, hc = m.predict_rew_end(frames[:, 3:4], act[:, 3:4], frames[:, 4:5], hc)
    path = os.path.join(OUT, "rew_end_wide.npz")
    np.savez_compressed(path, weights_checksum=np.float64(O.state_checksum(sd)), frames=frames.numpy(), act=act.numpy(),
                        burn_rew=br.numpy(), burn_end=be.numpy(), step3_rew=sr.numpy(), step3_end=se.numpy(),
                        hx=hc[0].numpy(), cx=hc[1].numpy())
    print("rew_end_wide logits rms", float(br.pow(2).mean().sqrt()), "size", os.path.getsize(path))


if __name__ == "__main__":
    ns = ref_import.load()
    torch.set_num_threads(8)
    make_denoiser_wide(ns)
    make_rew_end_wide(ns)
