"""WorldModelEnv under the reference trainer's default `training.compile_wm: True`: predict_next_obs and predict_rew_end wrapped
in torch.compile(..., mode="reduce-overhead") as trainer.py:178-184 builds them, on the default nets at 32 environments.

* parity: two actor-critic updates of 15 steps through ImaginationLoop, compiled against eager, with every environment
  truncated mid-rollout (reset_dead and burn-in run) -- frames, reward/termination logits, hx and cx bit-identical, loss and
  gradients within 1e-6;
* whole graphs: both methods compile with fullgraph=True, no cudagraph skips, and replayed steps launch nothing natively
  (the native work comes from the recorded graphs);
* weights are live: after a native AdamW step, load_state_dict or a replaced Parameter, the next replay equals an eager call
  with the new weights;
* eager unchanged: the launch counts of sample_ring and predict_rew_end are the parent build's."""
import random
import types

import pytest
import torch

gpu = pytest.mark.gpu

ENVS, HORIZON, ENV_HORIZON = 32, 15, 7   # every env is truncated at step 7 and 14: reset_dead + burn-in inside each update
# kernels one eager call launches on the default nets at 32 envs, 64 x 64, 3 Euler steps (parent build, weights already packed)
SAMPLE_RING_LAUNCHES = 329
PREDICT_REW_END_LAUNCHES = 58


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _world(dev, env_horizon=ENV_HORIZON, compiled=False, fullgraph=False):
    """bench.py's imagination block (cfg 3): denoiser, reward/termination model and policy, an in-memory loader; compiled the
    way trainer.py:182-184 does it."""
    from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig, ActorCriticLossConfig
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, DiffusionSamplerConfig, InnerModelConfig
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    rem = RewEndModel(RewEndModelConfig(512, 3, 64, 128, [2, 2, 2, 2], [32] * 4, [0] * 4, 4))
    randomize_module_(rem, 2025)
    ac = ActorCritic(ActorCriticConfig(512, 3, 64, [32, 32, 64, 64], [1, 1, 1, 1], 4))
    randomize_module_(ac, 2026)
    den, rem, ac = den.to(dev).eval(), rem.to(dev).eval(), ac.to(dev).train()
    with torch.no_grad():
        last = [m for m in rem.modules() if isinstance(m, torch.nn.Linear)][-1]
        last.weight[3].fill_(0.05); last.weight[4].fill_(-0.05)
    pool = [frame_stacks(ENVS, 4, 3, 64, 64, 4, 1000 + k)[:2] for k in range(8)]

    class Loader:
        batch_sampler = types.SimpleNamespace(batch_size=ENVS)

        def __iter__(self):
            k = 0
            while True:
                obs, act = pool[k % len(pool)]
                k += 1
                yield types.SimpleNamespace(obs=obs, act=act)

    env = WorldModelEnv(den, rem, Loader(), WorldModelEnvConfig(env_horizon, 4, DiffusionSamplerConfig(3)))
    if compiled:
        kw = dict(mode="reduce-overhead", fullgraph=fullgraph)
        env.predict_next_obs = torch.compile(env.predict_next_obs, **kw)
        env.predict_rew_end = torch.compile(env.predict_rew_end, **kw)
    ac.setup_training(env, ActorCriticLossConfig(HORIZON, 0.985, 0.95, 1.0, 0.001))
    return env, den, rem, ac


def _spy(env):
    """Records every step's frame, reward/termination logits, hx and cx.  The logits are taken inside predict_rew_end (the
    spy is traced into the compiled graph) and cloned after the step, before a later replay can overwrite them."""
    rem, seen, rec = env.rew_end_model, [], []
    real_predict = rem.predict_rew_end

    def predict(*a, **k):
        out = real_predict(*a, **k)
        seen.append(torch.cat([out[0], out[1]], -1))
        return out
    rem.predict_rew_end = predict
    real_step = env.step

    def step(act):
        out = real_step(act)
        rec.append([out[0].clone(), *[s.clone() for s in seen], env.hx_rew_end.clone(), env.cx_rew_end.clone()])
        seen.clear()
        return out
    env.step = step
    return rec


@pytest.fixture(autouse=True)
def _eager_random():
    """Random ops inside the compiled graphs (the sampler's noise, the Categorical draws) use torch's eager kernels, so that
    compiled and eager runs draw the same numbers."""
    import torch._inductor.config as ic

    with ic.patch(fallback_random=True):
        yield


def _updates(dev, compiled, n=2):
    torch._dynamo.reset()
    random.seed(7)
    torch.manual_seed(7)
    env, den, rem, ac = _world(dev, compiled=compiled)
    rec = _spy(env)
    losses, grads = [], []
    for _ in range(n):
        for p in ac.parameters():
            p.grad = None
        loss, _ = ac()
        loss.backward()
        losses.append(loss.detach().clone())
        grads.append(torch.cat([p.grad.reshape(-1) for p in ac.parameters()]))
    torch.cuda.synchronize()
    return rec, losses, grads


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


@gpu
def test_compiled_rollout_matches_eager_bit_for_bit():
    dev = _dev()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        eager = _updates(dev, compiled=False)
        comp = _updates(dev, compiled=True)
    finally:
        torch.use_deterministic_algorithms(prev)
    rec_e, loss_e, grad_e = eager
    rec_c, loss_c, grad_c = comp
    assert len(rec_e) == len(rec_c) == 2 * HORIZON
    for t, (a, b) in enumerate(zip(rec_e, rec_c)):
        assert len(a) == len(b), t
        for x, y in zip(a, b):
            assert torch.equal(x, y), f"step {t}: compiled differs from eager"
    for a, b in zip(loss_e, loss_c):
        assert _rel(b, a) <= 1e-6
    for a, b in zip(grad_e, grad_c):
        assert _rel(b, a) <= 1e-6


def _cycle(env, rounds):
    """`rounds` passes over every ring head of the two compiled methods, as env.step makes them (without deaths)."""
    t = env._frames.size(0)
    for _ in range(rounds * t):
        nxt, _ = env.predict_next_obs()
        env.predict_rew_end(nxt.unsqueeze(1))
        env._head = (env._head + 1) % t


@gpu
def test_whole_graphs_and_no_native_host_calls_on_replay():
    from torch._dynamo.utils import counters

    from diamond_b200 import _lib

    dev = _dev()
    torch._dynamo.reset()
    counters.clear()
    env, *_ = _world(dev, env_horizon=1000, compiled=True, fullgraph=True)
    env.reset()
    _cycle(env, 3)                       # warm-up, record, first replays of every ring head
    torch.cuda.synchronize()
    assert counters["inductor"]["cudagraph_skips"] == 0, dict(counters["inductor"])
    lib = _lib.lib()
    before = lib.dmd_launch_count(0)
    _cycle(env, 2)
    torch.cuda.synchronize()
    assert lib.dmd_launch_count(0) == before, "a replayed step made native host calls"
    assert counters["inductor"]["cudagraph_skips"] == 0


def _state(env):
    # the carried LSTM state's buffers themselves too: an eager predict_rew_end rebinds them, a compiled one writes them in place
    return (env._frames.clone(), env._acts.clone(), env._head, env.hx_rew_end, env.cx_rew_end, env.hx_rew_end.clone(),
            env.cx_rew_end.clone())


def _restore(env, s):
    env._frames.copy_(s[0]); env._acts.copy_(s[1]); env._head = s[2]
    env.hx_rew_end, env.cx_rew_end = s[3], s[4]
    env.hx_rew_end.copy_(s[5]); env.cx_rew_end.copy_(s[6])


def _call(env, fns, s):
    """One predict_next_obs + predict_rew_end from state `s`: (new frame, trajectory, hx, cx).  The sampler's noise is fixed
    (see _fixed_noise); the sampled reward and termination are left out, so nothing here depends on the RNG."""
    _restore(env, s)
    nxt, traj = fns[0]()
    fns[1](nxt.unsqueeze(1))
    out = [nxt.clone(), torch.stack(list(traj)).clone(), env.hx_rew_end.clone(), env.cx_rew_end.clone()]
    torch.cuda.synchronize()
    return out


def _fixed_noise(env, dev):
    noise = torch.randn(ENVS, 3, 64, 64, generator=torch.Generator(device=dev).manual_seed(5), device=dev)
    env.sampler._draw_noise = lambda buf: buf["traj"][0].copy_(noise)


@gpu
def test_replays_use_live_weights():
    from diamond_b200.envs import WorldModelEnv
    from diamond_b200.optim import AdamW

    dev = _dev()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        torch._dynamo.reset()
        env, den, rem, _ = _world(dev, env_horizon=1000, compiled=True)
        _fixed_noise(env, dev)
        env.reset()
        _cycle(env, 3)
        s = _state(env)
        compiled = (env.predict_next_obs, env.predict_rew_end)
        eager = (lambda: WorldModelEnv.predict_next_obs(env), lambda o: WorldModelEnv.predict_rew_end(env, o))
        before = _call(env, compiled, s)
        assert all(torch.equal(a, b) for a, b in zip(before, _call(env, eager, s)))

        saved = ({k: v.clone() for k, v in den.state_dict().items()}, {k: v.clone() for k, v in rem.state_dict().items()})
        params = list(den.parameters()) + list(rem.parameters())
        g = torch.Generator(device=dev).manual_seed(3)
        for p in params:
            p.grad = torch.randn(p.shape, generator=g, device=dev) * 1e-2
        AdamW(params, lr=1e-3).step()
        stepped = _call(env, compiled, s)
        assert all(torch.equal(a, b) for a, b in zip(stepped, _call(env, eager, s)))
        assert not torch.equal(stepped[0], before[0]) and not torch.equal(stepped[2], before[2])

        den.load_state_dict(saved[0]); rem.load_state_dict(saved[1])
        loaded = _call(env, compiled, s)
        assert all(torch.equal(a, b) for a, b in zip(loaded, before))

        with torch.no_grad():   # a replaced Parameter: refresh_weights() as for eager use, then the graphs re-record
            rem.head[0].weight = torch.nn.Parameter(rem.head[0].weight * 1.5)
            den.inner_model.conv_in.weight = torch.nn.Parameter(den.inner_model.conv_in.weight * 1.5)
        rem.refresh_weights(); den.inner_model.refresh_weights()
        want = _call(env, eager, s)
        got = _call(env, compiled, s)
        assert all(torch.equal(a, b) for a, b in zip(got, want))
        assert not torch.equal(got[0], before[0]) and not torch.equal(got[2], before[2])
    finally:
        torch.use_deterministic_algorithms(prev)


@gpu
def test_eager_launch_counts_unchanged():
    from diamond_b200 import _lib

    dev = _dev()
    env, *_ = _world(dev, env_horizon=1000)
    env.reset()
    _cycle(env, 1)                       # handles, packs and the sampler's own graphs exist
    lib = _lib.lib()
    n0 = lib.dmd_launch_count(0)
    nxt, _ = env.predict_next_obs()      # one sample_ring
    n1 = lib.dmd_launch_count(0)
    env.predict_rew_end(nxt.unsqueeze(1))
    n2 = lib.dmd_launch_count(0)
    assert (n1 - n0, n2 - n1) == (SAMPLE_RING_LAUNCHES, PREDICT_REW_END_LAUNCHES)
