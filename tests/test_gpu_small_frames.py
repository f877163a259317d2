"""GPU: frames smaller than 64 x 64 on the default 4-level nets (deepest level 4 x 4 to 7 x 7), a 5-level U-Net at 64 x 64, and
actor-critics whose levels are odd.

- dmd_attn_bwd at L = 1 .. 64 tokens (C = 32, 64) against float64 autograd, the parameter gradients added onto pre-filled buffers
  (as tests/test_gpu_backward_ops.py::test_attn_bwd does at L = 64).
- The default denoiser and its Euler sampler at 32 x 32, 40 x 40 and 32 x 64 against the reference's own outputs
  (tests/golden/denoiser_{32x32,40x40,32x64}.npz, oracle/make_golden_small_frames.py), with the checks of tests/test_gpu_denoiser.py.
- Training against the float64 oracle within the fp16-operand emulation's bounds (tests/test_gpu_training_configs.py): the
  default denoiser at 32 and 40, 128-channel attention (the split backward, attn_core_bwd_kernel) over 16, 25, 36 and 49 tokens,
  the 5-level U-Net at 64 x 64, the reward / termination model at 32 and 40, and the default actor-critic at img_size 40 and 84
  (floor max-pooling of the 5 x 5 and 21 x 21 levels) through its imagined rollout.
- The actor-critic's forward and its BPTT gradient at img_size 40 and 84 against the reference (tests/golden/actor_critic_small.npz).
- A 15-step WorldModelEnv rollout at 32 x 32 against the oracle's sampler on the same frame stacks.
- Denoising and training at 40 x 40 on poisoned workspaces (tests/test_gpu_poisoned_buffers.py's pattern)."""
import importlib.util
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import make_golden_small_frames as SF
from oracle import torch_oracle as O
from oracle import training_configs as TC

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _load(name):
    """A sibling test module by file (its helpers; the module is not a package)."""
    spec = importlib.util.spec_from_file_location(f"_small_frames_{name}", os.path.join(HERE, name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


BO = _load("test_gpu_backward_ops")
TD = _load("test_gpu_denoiser")
TGC = _load("test_gpu_training_configs")
PB = _load("test_gpu_poisoned_buffers")


# ------------------------------------------------------------------------------------------------ attention backward, any L <= 64
@pytest.mark.parametrize("c", [32, 64])
@pytest.mark.parametrize("L", [1, 4, 16, 25, 36, 49, 64])
def test_attn_bwd_any_token_count(L, c):
    """g_x and the six parameter gradients over L tokens laid out as 1 x L; the parameter gradients are added (inv_scale = 1/2,
    g_out scaled by 2) to pre-filled buffers."""
    dev = _dev()
    from diamond_b200 import ops

    g = BO._gen(700 + L + c)
    b, gs = 3, 32
    x = torch.randn(b, 1, L, c, generator=g) * 1.5 + 0.2
    gout = torch.randn(b, 1, L, c, generator=g)
    w = lambda *s: torch.randn(*s, generator=g) / s[-1] ** 0.5  # noqa: E731
    gamma, beta = 1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g)
    wqkv, bqkv, wout, bout = w(3 * c, c), 0.1 * torch.randn(3 * c, generator=g), w(c, c), 0.1 * torch.randn(c, generator=g)
    ref = BO.ref_attn(*(t.to(dev) for t in (x, gout, gamma, beta, wqkv, bqkv, wout, bout)))
    pre = [(torch.randn(r.shape, generator=g) * float(r.std() if r.numel() > 1 else 1.0)).float().to(dev) for r in ref[1:]]
    pgrads = tuple(p.clone() for p in pre)
    gx = ops.attn_bwd(x.to(dev), BO._gn_stats(x, gs).to(dev), gamma.to(dev), beta.to(dev), wqkv.to(dev), bqkv.to(dev), wout.to(dev),
                      (2 * gout).to(dev), gs, pgrads, inv_scale=torch.tensor([0.5], device=dev))
    names = ["dgamma", "dbeta", "dwqkv", "dbqkv", "dwout", "dbout"]
    errs = {"gx": BO._rel(gx, 2 * ref[0])}
    errs.update({n: BO._acc_rel(p, q, r) for n, p, q, r in zip(names, pgrads, pre, ref[1:])})
    print(f"attn_bwd L={L} C={c}:", {k: f"{v:.2e}" for k, v in errs.items()})
    # at L = 1 softmax is 1: the q / k gradients are exactly zero and g_x, d gamma come only through v and the residual
    assert max(errs.values()) < BO.TOL, errs


def test_attn_bwd_refuses_more_than_64_tokens():
    dev = _dev()
    from diamond_b200 import _lib

    lib, p = _lib.lib(), 0x1000
    rc = lib.dmd_attn_bwd(*([p] * 15), None, 2, 65, 64, 32, 1e-5, None)
    assert rc != 0 and "attention backward" in lib.dmd_last_error().decode()
    del dev


# ------------------------------------------------------------------------------------------------ denoiser / sampler vs the reference
@pytest.fixture
def small_frame_cases(monkeypatch):
    monkeypatch.setattr(TD, "_cases", lambda: SF.SMALL_FRAME_CASES)


@pytest.mark.parametrize("name", list(SF.SMALL_FRAME_CASES))
def test_denoiser_matches_reference_golden_at_small_frames(golden_dir, name, small_frame_cases):
    TD.test_denoiser_matches_reference_golden(golden_dir, name)


@pytest.mark.parametrize("name", list(SF.SMALL_FRAME_CASES))
@pytest.mark.parametrize("graph", [False, True])
def test_sampler_matches_reference_golden_at_small_frames(golden_dir, name, graph, small_frame_cases):
    TD.test_sampler_matches_reference_golden(golden_dir, name, graph)


# ------------------------------------------------------------------------------------------------ training vs float64
_A128 = O.InnerCfg(depths=[1, 1, 1, 1], channels=[32, 32, 64, 128])                      # mid attention at C = 128
_ONE128 = O.InnerCfg(cond_channels=64, depths=[1], channels=[128], attn_depths=[1])     # attention in every block, C = 128
DENOISER_CASES = dict(SF.SMALL_DENOISER_TRAIN, **{
    "A128_L16": dict(inner=_A128, h=32, w=32, b=2, seq=1, mask_off=[], wseed=7016, dseed=7017),
    "A128_L25": dict(inner=_A128, h=40, w=40, b=2, seq=1, mask_off=[], wseed=7025, dseed=7026),
    "A128_L36": dict(inner=_ONE128, h=6, w=6, b=3, seq=1, mask_off=[], wseed=7036, dseed=7037),
    "A128_L49": dict(inner=_ONE128, h=7, w=7, b=3, seq=1, mask_off=[], wseed=7049, dseed=7050),
    "A64_L36": dict(inner=O.InnerCfg(cond_channels=64, depths=[1], channels=[64], attn_depths=[1]), h=6, w=6, b=3, seq=1,
                    mask_off=[], wseed=7064, dseed=7065),
    # five levels at 64 x 64: the deepest is 4 x 4
    "U5_64": dict(inner=O.InnerCfg(depths=[1, 1, 1, 1, 1], channels=[64, 64, 64, 64, 64], attn_depths=[0, 0, 0, 0, 0]),
                  h=64, w=64, b=2, seq=1, mask_off=[], wseed=7105, dseed=7106),
})
REW_END_CASES = dict(SF.SMALL_REW_END_TRAIN, **{
    "R32": dict(cfg=O.RewEndCfg(img_size=32), b=4, T=5, death=(0, 2), pad=(3, 3), wseed=7132, dseed=7133),
})
ACTOR_CRITIC_CASES = {
    "AC40": dict(cfg=O.ActorCriticCfg(img_size=40), b=4, T=6, end=(2, 1), trunc=(4, 3), wseed=7140, dseed=7141),
    "AC84": dict(cfg=O.ActorCriticCfg(img_size=84), b=3, T=4, end=(1, 0), trunc=(2, 2), wseed=7184, dseed=7185),
}


@pytest.fixture
def small_training_cases(monkeypatch):
    for table, cases in ((TC.DENOISER_CASES, DENOISER_CASES), (TC.REW_END_CASES, REW_END_CASES),
                         (TC.ACTOR_CRITIC_CASES, ACTOR_CRITIC_CASES)):
        for k, v in cases.items():
            monkeypatch.setitem(table, k, v)


@pytest.mark.parametrize("name", list(DENOISER_CASES) + list(REW_END_CASES) + list(ACTOR_CRITIC_CASES))
def test_small_frame_training_matches_float64_oracle(name, small_training_cases):
    TGC._check_case(name, _dev())


# ------------------------------------------------------------------------------------------------ actor-critic vs the reference
@pytest.mark.parametrize("name", list(SF.SMALL_ACTOR_CRITIC))
def test_actor_critic_forward_and_bptt_match_reference(golden_dir, name):
    dev = _dev()
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig

    c = SF.SMALL_ACTOR_CRITIC[name]
    cfg = c["cfg"]
    g = np.load(os.path.join(golden_dir, "actor_critic_small.npz"))
    sd = O.seeded_actor_critic_state_dict(cfg, c["wseed"])
    assert abs(O.state_checksum(sd) - float(g[f"{name}_weights_checksum"])) < 1e-6 * abs(float(g[f"{name}_weights_checksum"]))
    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    ac.load_state_dict(sd)
    ac = ac.to(dev).train()
    obs, hx, cx, wl, wv = SF.actor_critic_inputs(c)
    logits, vals = [], []
    h, cc = hx.to(dev), cx.to(dev)
    for t in range(SF.AC_STEPS):
        o = ac.predict_act_value(obs[t].to(dev), (h, cc))
        logits.append(o.logits_act); vals.append(o.val); h, cc = o.hx_cx
    logits, vals = torch.stack(logits), torch.stack(vals)
    (logits * wl.to(dev)).sum().add((vals * wv.to(dev)).sum()).backward()
    torch.cuda.synchronize()
    errs = {k: TD._rel(v.detach().cpu(), torch.from_numpy(g[f"{name}_{k}"]))
            for k, v in (("logits", logits), ("val", vals), ("hx", h), ("cx", cc))}
    grads = dict(ac.named_parameters())
    keys = [str(k) for k in g[f"{name}_grad_keys"]]
    got = np.stack([grads[k].grad.detach().double().flatten().cpu()[torch.linspace(0, grads[k].numel() - 1, 16).round().long()].numpy()
                    for k in keys])
    ref = g[f"{name}_grad_samples"]
    norms = np.array([float(grads[k].grad.double().norm()) for k in keys])
    ref_norms = g[f"{name}_grad_norms"]
    e_norm = float(np.sqrt(((norms - ref_norms) ** 2).sum() / (ref_norms ** 2).sum()))
    e_samples = float(np.linalg.norm(got - ref) / np.linalg.norm(ref))
    print(f"{name}: forward {', '.join(f'{k} {v:.2e}' for k, v in errs.items())}; gradient norms {e_norm:.2e}, samples {e_samples:.2e}")
    assert max(errs.values()) < 1e-4, errs
    # the encoder's backward runs on fp16 operands (the float64 bounds of these shapes are in the training test above)
    assert e_norm < 5e-3 and e_samples < 1e-2, (e_norm, e_samples)


# ------------------------------------------------------------------------------------------------ imagined rollout at 32 x 32
def test_world_model_env_rollout_at_32x32_matches_oracle():
    """15 WorldModelEnv steps at 32 x 32 on the default net: every next frame equals the oracle's sample() on the same frame
    stack, actions and initial noise, up to quantiser-bucket flips."""
    dev = _dev()
    from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.diffusion import DiffusionSamplerConfig

    inner = O.InnerCfg()
    den, _ = TD._build(inner, 3232, dev)
    b, hw = 4, 32

    class RewEnd:
        def predict_rew_end(self, obs, act, next_obs, hx_cx=None):
            n, t = obs.shape[:2]
            hx = torch.zeros(1, n, 8, device=obs.device) if hx_cx is None else hx_cx[0] + 1
            return torch.zeros(n, t, 3, device=obs.device), torch.tensor([4.0, -4.0], device=obs.device).expand(n, t, 2), (hx, hx.clone())

    class Loader:
        batch_sampler = SimpleNamespace(batch_size=b)

        def __iter__(self):
            g = torch.Generator().manual_seed(1)
            while True:
                yield SimpleNamespace(obs=torch.rand(b, 4, 3, hw, hw, generator=g) * 2 - 1, act=torch.randint(0, 4, (b, 4), generator=g))

    env = WorldModelEnv(den, RewEnd(), Loader(), WorldModelEnvConfig(15, 2, DiffusionSamplerConfig(3)))
    cfg = O.DenoiserCfg(inner=inner)
    sd = {k: v.detach().cpu() for k, v in den.inner_model.state_dict().items()}
    obs0, _ = env.reset()
    assert obs0.shape == (b, 3, hw, hw)
    worst = 0.0
    for step in range(15):
        before_obs, before_act = env.obs_buffer.clone(), env.act_buffer.clone()
        act = torch.randint(0, 4, (b,), generator=torch.Generator().manual_seed(step)).to(dev)
        x0 = torch.randn(b, 3, hw, hw, generator=torch.Generator().manual_seed(200 + step))
        orig = torch.randn
        torch.randn = lambda *a, **k: x0.to(dev)
        try:
            obs, rew, end, trunc, info = env.step(act)
        finally:
            torch.randn = orig
        before_act[:, -1] = act
        with torch.no_grad():
            want, _ = O.sample(before_obs.cpu(), before_act.cpu(), x0, sd, cfg, O.SamplerCfg(3))
        alive = ~torch.logical_or(end, trunc).bool().cpu()
        if alive.any():
            d = (obs.cpu()[alive] - want[alive]).abs()
            worst = max(worst, float((d > 1e-3).float().mean()))
            assert float(d.max()) <= 3 * 2 / 255 + 1e-5
            assert float((d > 1e-3).float().mean()) < 0.08
        assert torch.equal(trunc.cpu(), torch.full((b,), int(step == 14)))
    print(f"WorldModelEnv 32x32: worst share of pixels off by > 1e-3 over 15 steps {worst:.2e}")


# ------------------------------------------------------------------------------------------------ poisoned workspaces
@PB.BYTES
@pytest.mark.parametrize("b,h,w", [(3, 40, 40), (2, 32, 64)])
def test_denoise_at_small_frames_on_poisoned_memory(b, h, w, byte):
    PB.test_denoise_and_inner_model_on_poisoned_memory("default", b, h, w, byte)


def _training_at_40(byte, dev):
    """Denoiser.forward (two autoregressive steps) + backward on the default net at 40 x 40, scratch and allocations poisoned."""
    den, i = PB._denoiser("default", dev)
    den.train()
    im = den.inner_model
    b, T = 3, i.num_steps_conditioning + 2
    obs = PB._levels((b, T, i.img_channels, 40, 40), 11, dev).float().div(255).mul(2).sub(1)
    act = torch.randint(0, i.num_actions, (b, T), generator=torch.Generator().manual_seed(12)).to(dev)
    batch = SimpleNamespace(obs=obs, act=act, mask_padding=torch.ones(b, T, dtype=torch.bool, device=dev))
    PB.poison_scratch(byte, im)
    torch.manual_seed(5)
    with PB.poisoned_allocations(byte):
        loss, _ = den(batch)
        loss.backward()
        out = {"loss": loss.detach().reshape(1), "grad": torch.cat([p.grad.reshape(-1) for p in den.parameters()])}
    torch.cuda.synchronize()
    return out


@PB.BYTES
def test_denoiser_training_at_40x40_on_poisoned_memory(byte):
    dev = _dev()
    ref, again = _training_at_40(None, dev), _training_at_40(None, dev)
    PB._check_close(f"denoiser training 40x40 0x{byte:02X}", _training_at_40(byte, dev), ref, again)
