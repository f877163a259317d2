"""Records what the UNMODIFIED reference computes for the CPU tests that compare the mirror / oracle with it, so that those
tests run without the reference tree:

    DIAMOND_REFERENCE_SRC=<reference checkout>/src python oracle/make_reference_records.py

writes tests/golden/reference_records.npz: tensors compared with a tolerance or bit for bit, and under the key "records" a
JSON document with the state-dict layouts, the optimizer's parameter split and SHA-256 digests of the long bit-exact
WorldModelEnv / env-loop streams.  The inputs are the ones the tests build (seeded); the tests recompute the
mirror / oracle side live.
"""
import hashlib
import importlib.util
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# inputs shared with the tests (tests/test_oracle_vs_reference.py, tests/test_host_logic.py)
DENOISE_INNER = dict(depths=[1, 1, 1], channels=[32, 32, 64], attn_depths=[0, 1, 0], cond_channels=64, num_actions=5)
EDM_INNER = (3, 2, 64, [1, 1], [32, 32], [0, 0], 4)
EDM_SIGMA_DISTRIBUTION = (-0.4, 1.2, 2e-3, 20)
LAYOUT_INNERS = {
    "default": O.InnerCfg(),
    "small": O.InnerCfg(depths=[1, 2, 1], channels=[32, 64, 32], attn_depths=[0, 0, 1], cond_channels=64,
                        num_steps_conditioning=2, num_actions=6),
}


def digest(t: torch.Tensor) -> list:
    """(dtype, shape, sha256 of the bytes): equal digests <=> torch.equal for tensors of one dtype."""
    return [str(t.dtype), list(t.shape), hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()]


def edm_x() -> torch.Tensor:
    return torch.rand(5, 3, 16, 16, generator=torch.Generator().manual_seed(0)) * 2 - 1


def edm_pieces(den, sigma_distribution_config, x):
    den.setup_training(sigma_distribution_config(*EDM_SIGMA_DISTRIBUTION))
    torch.manual_seed(123)
    sigma = den.sample_sigma_training(5, torch.device("cpu"))
    noisy = den.apply_noise(x, sigma, 0.3)
    cs = den.compute_conditioners(sigma)
    model_out = torch.randn(5, 3, 16, 16)
    wrapped = den.wrap_model_output(noisy, model_out, cs)
    s0 = den.compute_conditioners(torch.tensor(1.7))   # 0-dim sigma, as DiffusionSampler passes it (diffusion_sampler.py:44)
    return {"sigma": sigma, "noisy": noisy, "c_in": cs.c_in, "c_out": cs.c_out, "c_skip": cs.c_skip, "c_noise": cs.c_noise,
            "wrapped": wrapped, **{"s0_" + k: v for k, v in vars(s0).items()}}


def _test_module(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    torch.set_num_threads(8)
    ns = ref_import.load()
    D = ns.diffusion
    arrays, records = {}, {}

    # oracle restatement of Denoiser.denoise / compute_model_output
    inner = O.InnerCfg(**DENOISE_INNER)
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), 31337)
    den = D.Denoiser(D.DenoiserConfig(D.InnerModelConfig(3, 4, 64, inner.depths, inner.channels, inner.attn_depths,
                                                         inner.num_actions), 0.5, 0.3)).eval()
    den.inner_model.load_state_dict(sd)
    obs, act, x = O.synthetic_inputs(3, inner, 32, 32, 9)
    sig = torch.tensor([0.01, 0.5, 7.0])
    with torch.no_grad():
        arrays["denoise"] = den.denoise(x, sig, obs.reshape(3, 12, 32, 32), act).numpy()
        cs = den.compute_conditioners(sig)
        arrays["model_output"] = den.compute_model_output(x, obs.reshape(3, 12, 32, 32), act, cs).numpy()

    # host-side EDM pieces of the training forward
    ref = D.Denoiser(D.DenoiserConfig(D.InnerModelConfig(*EDM_INNER), 0.5, 0.3))
    for k, v in edm_pieces(ref, D.SigmaDistributionConfig, edm_x()).items():
        arrays["edm_" + k] = v.numpy()

    # state-dict layouts and the optimizer's weight-decay split of the mirror (utils.configure_opt, utils.py:129-166)
    records["state_dict_layout"] = {}
    for key, ic in LAYOUT_INNERS.items():
        r = D.Denoiser(D.DenoiserConfig(D.InnerModelConfig(ic.img_channels, ic.num_steps_conditioning, ic.cond_channels,
                                                           list(ic.depths), list(ic.channels), list(ic.attn_depths),
                                                           ic.num_actions), 0.5, 0.3))
        records["state_dict_layout"][key] = [[k, list(v.shape)] for k, v in r.state_dict().items()]
    host_logic = _test_module("test_host_logic")
    mirror = host_logic._denoiser(O.InnerCfg())
    names = {id(p): n for n, p in mirror.named_parameters()}
    opt = ns.utils.configure_opt(mirror, 1e-4, 1e-2, 1e-8)
    records["configure_opt_groups"] = [[names[id(p)] for p in g["params"]] for g in opt.param_groups]

    # WorldModelEnv and env loop driven by the fakes of tests/test_env_host_logic.py
    env_logic = _test_module("test_env_host_logic")
    ref_env = ns.envs.world_model_env
    records["world_model_env"] = [digest(t) for t in env_logic._run_env(ref_env, ref_env.WorldModelEnvConfig, D.DiffusionSamplerConfig(3))]
    records["env_loop"] = [digest(t) for t in env_logic._run_loop(ns.env_loop.make_env_loop, ref_env, ref_env.WorldModelEnvConfig,
                                                                  D.DiffusionSamplerConfig(3))]
    rew, end, trunc, vb = env_logic.lambda_returns_inputs()
    records["lambda_returns"] = {str(lam): digest(ns.actor_critic.compute_lambda_returns(rew, end, trunc, vb, 0.985, lam))
                                 for lam in env_logic.LAMBDAS}

    np.savez_compressed(os.path.join(OUT, "reference_records.npz"), records=np.array(json.dumps(records)), **arrays)


def load_records(golden_dir):
    """The JSON part of tests/golden/reference_records.npz."""
    with np.load(os.path.join(golden_dir, "reference_records.npz")) as z:
        return json.loads(str(z["records"]))


if __name__ == "__main__":
    main()
