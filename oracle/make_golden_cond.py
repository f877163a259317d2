"""Generates the fixtures of nets with conditioning vectors wider than 256 channels (tests/golden/denoiser_cond2048.npz,
rew_end_cond512.npz) by running the UNMODIFIED reference (imported as oracle/make_golden.py does) on seeded inputs and
seeded 'de-zeroed' weights:

    DIAMOND_REFERENCE_SRC=<reference checkout>/src python oracle/make_golden_cond.py

denoiser_cond2048: a [64, 128, 128, 128] U-Net with cond_channels = 2048 (a 7168 x 2048 FiLM table, a 2048 -> 2048 cond MLP,
512-wide action embeddings): model output, denoised frame, an Euler sampler trajectory, and Denoiser.forward + backward over
two autoregressive steps with one padded target (loss and gradient summary, its draws replayed).
rew_end_cond512: the default reward / termination encoder with cond_channels = 512: a 3-step burn-in call, one step carrying
the LSTM state, and RewEndModel.forward + backward over segments with a death and a padded tail (loss and gradient summary).

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

# inference and training share the net: training draws and batch follow training_configs.denoiser_inputs
DENOISER_COND = dict(
    inner=O.InnerCfg(cond_channels=2048, depths=[1, 1, 1, 1], channels=[64, 128, 128, 128]), h=64, w=64, b=2, wseed=2049,
    iseed=82, sigmas=[0.7, 3.0], sampler=O.SamplerCfg(num_steps_denoising=3), rng_seed=9,
    train=dict(b=2, seq=2, mask_off=[(1, 5)], dseed=2050),
)
REW_END_COND = dict(cfg=O.RewEndCfg(cond_channels=512), wseed=2051, dseed=2052, b=2,
                    train=dict(b=4, T=7, death=(1, 3), pad=(2, 5), dseed=2053))


def denoiser_train_case(c=DENOISER_COND):
    """The training case of c in the layout of training_configs.DENOISER_CASES."""
    t = c["train"]
    return dict(inner=c["inner"], h=c["h"], w=c["w"], b=t["b"], seq=t["seq"], mask_off=t["mask_off"], wseed=c["wseed"], dseed=t["dseed"])


def rew_end_train_case(c=REW_END_COND):
    """The training case of c in the layout of training_configs.REW_END_CASES."""
    t = c["train"]
    return dict(cfg=c["cfg"], b=t["b"], T=t["T"], death=t["death"], pad=t["pad"], wseed=c["wseed"], dseed=t["dseed"])


def rew_end_predict_inputs(c=REW_END_COND):
    cfg, b = c["cfg"], c["b"]
    rng = np.random.default_rng(c["dseed"])
    frames = torch.from_numpy(rng.integers(0, 256, size=(b, 5, cfg.img_channels, cfg.img_size, cfg.img_size)).astype(np.float32))
    frames = frames.div(255).mul(2).sub(1)
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, 4)).astype(np.int64))
    return frames, act


def _summary(named):
    grads = [(k, p.grad) for k, p in named]
    assert all(g is not None for _, g in grads)
    return O.grad_summary(grads)


def make_denoiser_cond(ns):
    from oracle.make_golden import build_reference

    c = DENOISER_COND
    inner = c["inner"]
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    den = build_reference(ns, inner, sd)
    obs, act, x_noisy = O.synthetic_inputs(c["b"], inner, c["h"], c["w"], c["iseed"])
    sig = torch.tensor(c["sigmas"], dtype=torch.float32)
    b, t, ch, h, w = obs.shape
    s = c["sampler"]
    assert s.order == 1 and s.s_churn == 0   # the sampler draws only x0
    with torch.no_grad():
        cs = den.compute_conditioners(sig)
        mo = den.compute_model_output(x_noisy, obs.reshape(b, t * ch, h, w), act, cs)
        dn = den.wrap_model_output(x_noisy, mo, cs)
        sampler = ns.diffusion.DiffusionSampler(den, ns.diffusion.DiffusionSamplerConfig(
            s.num_steps_denoising, s.sigma_min, s.sigma_max, s.rho, s.order, s.s_churn, s.s_tmin, s.s_tmax, s.s_noise))
        torch.manual_seed(c["rng_seed"])
        x, traj = sampler.sample(obs, act)

    # training: Denoiser.forward + backward, the standard-normal draws of training_configs.denoiser_inputs replayed
    D = ns.diffusion
    tc = denoiser_train_case()
    den = build_reference(ns, inner, sd).train()
    sc = O.SigmaDistCfg()
    den.setup_training(D.SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    tobs, tact, mask, draws = TC.denoiser_inputs(tc)
    tb, T = tobs.shape[:2]
    batch = ns.data.Batch(obs=tobs.clone(), act=tact, rew=torch.zeros(tb, T), end=torch.zeros(tb, T, dtype=torch.long),
                          trunc=torch.zeros(tb, T, dtype=torch.long), mask_padding=mask, info=[{}] * tb, segment_ids=[None] * tb)
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

    path = os.path.join(OUT, "denoiser_cond2048.npz")
    np.savez_compressed(path, weights_checksum=np.float64(O.state_checksum(sd)), sigmas_in=sig.numpy(), model_output=mo.numpy(),
                        denoised=dn.numpy(), sampler_sigmas=sampler.sigmas.numpy(), x0=traj[0].numpy(), sample_x=x.numpy(),
                        trajectory=torch.stack(traj).numpy(),
                        train_inputs_checksum=np.float64(TC.inputs_checksum([tobs, tact, mask] + q_all(draws))),
                        train_loss=np.float64(loss.item()), grad_keys=np.array(keys), grad_norms=norms, grad_samples=samples)
    print("denoiser_cond2048 model_output rms", float(mo.pow(2).mean().sqrt()), "loss", loss.item(), "size", os.path.getsize(path))


def q_all(draws):
    return [t for s in draws for t in s]


def make_rew_end_cond(ns):
    c = REW_END_COND
    cfg = c["cfg"]
    R = ns.rew_end_model
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"])

    def model():
        m = R.RewEndModel(R.RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                              list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
        assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == O.rew_end_shapes(cfg)
        m.load_state_dict(sd)
        return m

    m = model().eval()
    frames, act = rew_end_predict_inputs()
    with torch.no_grad():
        br, be, hc = m.predict_rew_end(frames[:, 0:3], act[:, 0:3], frames[:, 1:4])
        sr, se, hc = m.predict_rew_end(frames[:, 3:4], act[:, 3:4], frames[:, 4:5], hc)

    m = model().train()
    obs, tact, rew, end, mask, final_obs = TC.rew_end_inputs(rew_end_train_case())
    b = obs.size(0)
    info = [{"final_observation": final_obs[i]} if i in final_obs else {} for i in range(b)]
    batch = ns.data.Batch(obs=obs.clone(), act=tact, rew=rew, end=end, trunc=torch.zeros_like(end), mask_padding=mask, info=info,
                          segment_ids=[None] * b)
    loss, metrics = m(batch)
    loss.backward()
    keys, norms, samples = _summary(m.named_parameters())

    path = os.path.join(OUT, "rew_end_cond512.npz")
    np.savez_compressed(path, weights_checksum=np.float64(O.state_checksum(sd)), frames=frames.numpy(), act=act.numpy(),
                        burn_rew=br.numpy(), burn_end=be.numpy(), step3_rew=sr.numpy(), step3_end=se.numpy(),
                        hx=hc[0].numpy(), cx=hc[1].numpy(),
                        train_inputs_checksum=np.float64(TC.inputs_checksum([obs, tact, rew, end, mask] + list(final_obs.values()))),
                        train_loss=np.float64(loss.item()), loss_rew=np.float64(metrics["loss_rew"].item()),
                        loss_end=np.float64(metrics["loss_end"].item()), grad_keys=np.array(keys), grad_norms=norms,
                        grad_samples=samples)
    print("rew_end_cond512 logits rms", float(br.pow(2).mean().sqrt()), "loss", loss.item(), "size", os.path.getsize(path))


if __name__ == "__main__":
    from oracle import ref_import

    ns = ref_import.load()
    torch.set_num_threads(8)
    make_denoiser_cond(ns)
    make_rew_end_cond(ns)
