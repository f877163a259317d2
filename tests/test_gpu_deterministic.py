"""Deterministic mode: with torch.use_deterministic_algorithms(True) every native call is bit-reproducible.  Each case runs
twice and compares bytes; the second run starts from poisoned cached workspaces and runs beside a bounded load on another
stream, so its CTAs are scheduled and finish in another order.  The accuracy checks of the existing suite run again in the
mode against the same references and bounds."""
import contextlib
import os

# torch's own cuBLAS calls refuse deterministic mode without a fixed workspace configuration; it is read when cuBLAS starts
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import numpy as np  # noqa: E402
import pytest  # noqa: E402
import torch  # noqa: E402

import test_gpu_denoiser as TD  # noqa: E402
import test_gpu_imagination_models as TI  # noqa: E402
import test_gpu_poisoned_buffers as TP  # noqa: E402
import test_gpu_rew_end_training as TR  # noqa: E402
import test_gpu_training as TT  # noqa: E402
import test_gpu_training_configs as TGC  # noqa: E402
import test_gpu_uint8_frames as TU  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402
from oracle import training_configs as TC  # noqa: E402

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def deterministic():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


@contextlib.contextmanager
def busy(dev):
    """40 chained 2048² matmuls on a side stream (a few ms): they hold part of the SMs while the measured call runs."""
    s = torch.cuda.Stream(dev)
    a = torch.randn(2048, 2048, device=dev) / 64
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        for _ in range(40):
            a = torch.tanh(a @ a)
    try:
        yield
    finally:
        torch.cuda.synchronize()


@contextlib.contextmanager
def poisoned(dev, *modules):
    """The second run's conditions: the modules' cached scratch poisoned, every buffer the package allocates meanwhile
    poisoned, and the side-stream load running."""
    torch.cuda.synchronize()
    TP.poison_scratch(0xFF, *modules)
    with TP.poisoned_allocations(0xFF), busy(dev):
        yield


def twice(dev, run, *modules):
    """run() on a clean start, then again under `poisoned`; both results as CPU tensors."""
    with deterministic():
        first = [t.detach().cpu().clone() for t in run()]
        with poisoned(dev, *modules):
            second = [t.detach().cpu().clone() for t in run()]
    return first, second


def assert_bit_equal(label, a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and x.dtype == y.dtype
        assert torch.equal(x.view(torch.uint8) if x.is_floating_point() else x, y.view(torch.uint8) if y.is_floating_point() else y), \
            f"{label}: output {i} differs between two runs ({int((x != y).sum())} of {x.numel()} elements)"


def _grads(m):
    return [p.grad.detach() for _, p in m.named_parameters() if p.grad is not None]


def test_python_side_passes_torchs_flag():
    dev = TD._dev()
    den, _ = TD._build(O.InnerCfg(depths=[1, 1, 1, 1]), 5, dev)
    from diamond_b200 import _lib

    seen = []
    lib = _lib.lib()
    orig = lib.dmd_denoiser_set_deterministic

    class Spy:
        def __getattr__(self, k):
            return getattr(lib, k)

        def dmd_denoiser_set_deterministic(self, h, on):
            seen.append(on)
            return orig(h, on)

    import diamond_b200.utils as U
    real = U._lib.lib
    U._lib.lib = lambda: Spy()
    try:
        den.inner_model._native()
        with deterministic():
            den.inner_model._native()
        den.inner_model._native()
    finally:
        U._lib.lib = real
    assert seen == [0, 1, 0]


def test_denoiser_b32_forward_is_bit_reproducible():
    dev = TD._dev()
    inner = O.InnerCfg()
    den, _ = TD._build(inner, 2024, dev)
    obs, act, x0 = O.synthetic_inputs(32, inner, 64, 64, 100)
    flat = obs.reshape(32, -1, 64, 64).to(dev)
    sig = torch.linspace(0.002, 20.0, 32, device=dev)

    def run():
        return den._native_forward(x0.to(dev), sig, flat, act.to(dev), True, False)[:1]
    a, b = twice(dev, run, den.inner_model)
    assert_bit_equal("denoiser B=32", a, b)
    with deterministic():   # the bench.py workload against the float64-checked oracle, at the default mode's bounds
        TD.test_benchmarked_batch_sizes_match_the_oracle(32)


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("name", ["denoiser_default", "denoiser_small_heun", "denoiser_padded"])
def test_sampler_is_bit_reproducible(name, graph):
    dev = TD._dev()
    from diamond_b200.models.diffusion import DiffusionSampler, DiffusionSamplerConfig

    c = TD._cases()[name]
    den, _ = TD._build(c["inner"], c["wseed"], dev)
    s = c["sampler"]
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(s.num_steps_denoising, s.sigma_min, s.sigma_max, s.rho, s.order,
                                                           s.s_churn, s.s_tmin, s.s_tmax, s.s_noise))
    sampler.use_cuda_graph = graph
    obs, act, _ = O.synthetic_inputs(c["b"], c["inner"], c["h"], c["w"], c["iseed"])

    def run():
        torch.manual_seed(11)   # the initial noise and the churn draws
        outs = []
        for _ in range(2):   # with a graph, the second call replays it
            x, traj = sampler.sample(obs.to(dev), act.to(dev))
            outs += [x] + list(traj)
        return outs
    a, b = twice(dev, run, den.inner_model)
    assert_bit_equal(f"sample() {name} graph={graph}", a, b)


def test_mode_toggle_rebuilds_and_restores_the_sampler_plan():
    """Off -> on -> off on one sampler and workspace: the off results before and after are bit-identical (the plan and graph
    of the default mode are rebuilt as they were), and the on result is within the statistics' summation-order noise."""
    dev = TD._dev()
    from diamond_b200 import _lib
    from diamond_b200.models.diffusion import DiffusionSampler, DiffusionSamplerConfig

    inner = O.InnerCfg(depths=[1, 1, 1, 1])
    den, _ = TD._build(inner, 9, dev)
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(3))
    obs, act, x0 = O.synthetic_inputs(4, inner, 64, 64, 1)
    orig = torch.randn
    torch.randn = lambda *a, **k: x0.to(dev)
    try:
        def run():   # the first call of a mode captures a graph, the second replays it: its launch count is the graph's
            for _ in range(2):
                _lib.lib().dmd_launch_count(1)
                x, _ = sampler.sample(obs.to(dev), act.to(dev))
                torch.cuda.synchronize()
            return x.cpu().clone(), _lib.lib().dmd_launch_count(0)
        off1, n_off = run()
        with deterministic():
            on, n_on = run()
        off2, n_off2 = run()
    finally:
        torch.randn = orig
    assert torch.equal(off1.view(torch.uint8), off2.view(torch.uint8))
    assert n_off == n_off2 and n_on > n_off, (n_off, n_on, n_off2)
    assert float((on - off1).abs().max()) <= 2 / 255 + 1e-6


@pytest.mark.parametrize("name", ["denoiser_default_training", "denoiser_small_training"])
def test_training_step_is_bit_reproducible_and_accurate(golden_dir, name):
    """Loss and the whole gradient of Denoiser.forward (its autoregressive steps) + backward, twice; then the existing
    reference check of the step in the mode."""
    dev = TD._dev()
    from oracle.make_golden import CASES, TRAIN_CASES

    tc = TRAIN_CASES[name]
    c = CASES[tc["case"]]
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    draws = [tuple(torch.from_numpy(g[k][i]) for k in ("raw_sigma", "raw_offset", "raw_noise")) for i in range(tc["seq"])]
    obs, act, mask = (torch.from_numpy(g[k]) for k in ("obs", "act", "mask_padding"))
    sd = O.seeded_state_dict(O.inner_model_shapes(c["inner"]), c["wseed"])

    def run():
        loss, _, grads = TT._native_step(c["inner"], sd, obs, act, mask, draws, dev)
        return [torch.tensor([loss], dtype=torch.float64)] + list(grads.values())
    a, b = twice(dev, run)
    assert_bit_equal(name, a, b)
    with deterministic():
        TT.test_denoiser_training_step_matches_reference(golden_dir, name)


def _rew_end_twice(dev):
    cfg = O.RewEndCfg()
    inputs = TR._seeded_batch(32, 19, 1900)
    model = TR._model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 779), dev)

    def run():
        loss, _, logits = TR._native_step(model, TR._batch(*inputs, dev))
        return [loss.detach().reshape(1), logits[0], logits[1]] + _grads(model)
    return twice(dev, run, model)


def test_rew_end_training_is_bit_reproducible_and_accurate():
    dev = TD._dev()
    a, b = _rew_end_twice(dev)
    assert_bit_equal("rew_end 32 x 19", a, b)
    with deterministic():
        TR.test_rew_end_training_trainer_shape_matches_oracle()


def test_actor_critic_update_is_bit_reproducible_and_accurate(monkeypatch):
    dev = TD._dev()
    d = TI._bench_rollout_data()
    sd = O.seeded_actor_critic_state_dict(O.ActorCriticCfg(), TI.AC_SEED)
    runs = []
    for k in range(2):
        ac = TI._native_ac(sd, dev)
        with deterministic():
            if k:
                with poisoned(dev):
                    runs.append(TI._run_native_updates(ac, d, TI.AC_T, 1, monkeypatch, dev)[0])
            else:
                runs.append(TI._run_native_updates(ac, d, TI.AC_T, 1, monkeypatch, dev)[0])
    a, b = runs
    assert a["loss"] == b["loss"] and a["logs"] == b["logs"]
    assert_bit_equal("actor-critic logits / values", [a["logits"], a["val"]], [b["logits"], b["val"]])
    assert_bit_equal("actor-critic gradients", list(a["grads"].values()), list(b["grads"].values()))
    with deterministic():
        TI.test_actor_critic_benchmark_shape_two_updates_match_oracle(monkeypatch)


def test_world_model_env_rollout_is_bit_reproducible():
    """15 WorldModelEnv steps (native sampler + native reward / termination model), twice from the same seeds."""
    dev = TD._dev()
    from types import SimpleNamespace

    from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.diffusion import DiffusionSamplerConfig

    inner = O.InnerCfg(depths=[1, 1, 1, 1])
    den, _ = TD._build(inner, 77, dev)
    cfg = O.RewEndCfg()
    rew_end = TR._model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 779), dev).eval()

    class Loader:
        batch_sampler = SimpleNamespace(batch_size=8)

        def __iter__(self):
            g = torch.Generator().manual_seed(0)
            while True:
                yield SimpleNamespace(obs=torch.rand(8, 4, 3, 64, 64, generator=g) * 2 - 1, act=torch.randint(0, 4, (8, 4), generator=g))

    def run():
        torch.manual_seed(1234)
        env = WorldModelEnv(den, rew_end, Loader(), WorldModelEnvConfig(15, 2, DiffusionSamplerConfig(3)))
        obs, _ = env.reset()
        outs = [obs]
        for step in range(15):
            act = torch.randint(0, 4, (8,), generator=torch.Generator().manual_seed(step)).to(dev)
            obs, rew, end, trunc, _ = env.step(act)
            outs += [obs, rew, end, trunc]
        return outs
    a, b = twice(dev, run, den.inner_model, rew_end)
    assert_bit_equal("WorldModelEnv 15 steps", a, b)


def test_uint8_training_is_bit_reproducible():
    """The uint8 frame path of Denoiser.forward: loss and whole gradient, twice."""
    dev = TD._dev()
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig

    inner = O.InnerCfg(depths=[1, 1, 1, 1])
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), 31)
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths), inner.num_actions), 0.5, 0.3))
    den.inner_model.load_state_dict(sd)
    den = den.to(dev).train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    g = torch.Generator().manual_seed(3)
    obs = torch.randint(0, 256, (8, inner.num_steps_conditioning + 2, 3, 64, 64), generator=g, dtype=torch.uint8).to(dev)
    act = torch.randint(0, 4, (8, inner.num_steps_conditioning + 2), generator=g).to(dev)
    mask = torch.ones(8, inner.num_steps_conditioning + 2, dtype=torch.bool, device=dev)

    def run():
        torch.manual_seed(77)
        den.zero_grad(set_to_none=True)
        loss, _ = den(TT._Batch(obs, act, mask))
        loss.backward()
        return [loss.detach().reshape(1)] + _grads(den.inner_model)
    a, b = twice(dev, run, den.inner_model)
    assert_bit_equal("uint8 training", a, b)


def test_padded_84x84_inference_is_bit_reproducible():
    dev = TD._dev()
    inner = O.InnerCfg()
    den, _ = TD._build(inner, 2024, dev)
    obs, act, x0 = O.synthetic_inputs(4, inner, 84, 84, 100)
    flat = obs.reshape(4, -1, 84, 84).to(dev)
    sig = torch.linspace(0.1, 5.0, 4, device=dev)

    def run():
        return den._native_forward(x0.to(dev), sig, flat, act.to(dev), True, False)[:1]
    a, b = twice(dev, run, den.inner_model)
    assert_bit_equal("denoiser 84 x 84", a, b)


# Training cases in the shape of oracle/training_configs.py whose attention backward takes the split path only in this mode
# (C <= 64) below 8 x 8, whose 4 x 4 levels take their statistics from OP_STATS, and the [64, 128, 128, 128] net with
# attention at C = 128; two autoregressive steps each but the 6 x 6 case.  Accuracy: tests/test_gpu_training_configs.py's float64-autograd check
# with the fp16-operand emulation's bounds.
DET_TRAINING_CASES = {
    "DET32_C64": dict(inner=O.InnerCfg(depths=[1, 1, 1, 1], channels=[64, 64, 64, 64]), h=32, w=32, b=3, seq=2, mask_off=[],
                      wseed=9101, dseed=9102),
    "DET32_C32": dict(inner=O.InnerCfg(depths=[1, 1, 1, 1], channels=[32, 32, 32, 32], attn_depths=[0, 0, 0, 1]), h=32, w=32, b=3,
                      seq=2, mask_off=[], wseed=9103, dseed=9104),
    # tests/test_gpu_small_frames.py's A64_L36 (one step: at two, the emulation's own bound exceeds the harness's cap)
    "DET_L36_C64": dict(inner=O.InnerCfg(cond_channels=64, depths=[1], channels=[64], attn_depths=[1]), h=6, w=6, b=3, seq=1,
                        mask_off=[], wseed=7064, dseed=7065),
    "DET32_W128": dict(inner=O.InnerCfg(depths=[1, 1, 1, 1], channels=[64, 128, 128, 128], attn_depths=[0, 0, 0, 1]), h=32, w=32,
                       b=2, seq=2, mask_off=[], wseed=9107, dseed=9108),
}


@pytest.mark.parametrize("name", list(DET_TRAINING_CASES))
def test_split_attention_and_small_level_training_is_bit_reproducible_and_accurate(name, monkeypatch):
    dev = TD._dev()
    monkeypatch.setitem(TC.DENOISER_CASES, name, DET_TRAINING_CASES[name])

    def run():
        loss, grads = TGC._native(name, dev)
        return [torch.tensor([loss], dtype=torch.float64)] + [grads[k] for k in sorted(grads)]
    a, b = twice(dev, run)
    assert_bit_equal(name, a, b)
    with deterministic():
        TGC._check_case(name, dev)


def test_rew_end_predict_is_bit_reproducible():
    """predict_rew_end at 32 envs x 19 steps (inference plan), twice."""
    dev = TD._dev()
    cfg = O.RewEndCfg()
    model = TR._model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 779), dev).eval()
    g = torch.Generator().manual_seed(19)
    obs = (torch.rand(32, 19, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    nxt = (torch.rand(32, 19, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    act = torch.randint(0, 4, (32, 19), generator=g).to(dev)

    def run():
        with torch.no_grad():
            rew, end, (hx, cx) = model.predict_rew_end(obs, act, nxt)
        return [rew, end, hx, cx]
    a, b = twice(dev, run, model)
    assert_bit_equal("rew_end predict 32 x 19", a, b)


def test_world_model_env_with_uint8_loader_is_bit_reproducible():
    """The uint8 inference paths: WorldModelEnv over a uint8 loader (the pool, the initial-condition decode and the reward /
    termination burn-in on uint8 frames), 15 steps, twice."""
    dev = TD._dev()
    den, _ = TU._denoiser(dev, (1, 1, 1, 1))
    den.eval()
    rew_end, _ = TU._rew_end(dev)
    rew_end.eval()

    def run():
        env = TU._env(den, rew_end, True, dev)
        torch.manual_seed(0)
        obs, _ = env.reset()
        outs = [obs, env.hx_rew_end.clone(), env.cx_rew_end.clone()]
        for step in range(15):
            act = torch.randint(0, 4, (8,), device=dev)
            obs, rew, end, trunc, _ = env.step(act)
            outs += [obs, rew, end, trunc]
        return outs
    a, b = twice(dev, run, den.inner_model, rew_end)
    assert_bit_equal("WorldModelEnv uint8 loader", a, b)


def test_mode_toggle_between_training_steps_and_predict_calls():
    """The mode is part of the training-plan and encoder-plan keys: on, off, on over one pooled training workspace (and one
    reward / termination inference workspace) gives the first result again, bit for bit."""
    dev = TD._dev()
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig

    inner = O.InnerCfg(depths=[1, 1, 1, 1])
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths), inner.num_actions), 0.5, 0.3))
    den.inner_model.load_state_dict(O.seeded_state_dict(O.inner_model_shapes(inner), 41))
    den = den.to(dev).train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    g = torch.Generator().manual_seed(4)
    batch = TT._Batch((torch.rand(4, 5, 3, 64, 64, generator=g) * 2 - 1).to(dev), torch.randint(0, 4, (4, 5), generator=g).to(dev),
                      torch.ones(4, 5, dtype=torch.bool, device=dev))

    def step():
        torch.manual_seed(5)
        den.zero_grad(set_to_none=True)
        loss, _ = den(batch)
        loss.backward()
        torch.cuda.synchronize()
        return [loss.detach().cpu().reshape(1)] + [t.cpu().clone() for t in _grads(den.inner_model)]

    cfg = O.RewEndCfg()
    rem = TR._model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 42), dev).eval()
    obs = (torch.rand(8, 3, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    act = torch.randint(0, 4, (8, 3), generator=g).to(dev)

    def predict():
        with torch.no_grad():
            return [t.cpu().clone() for t in rem.predict_rew_end(obs, act, obs)[:2]]

    with deterministic():
        on1, p1 = step(), predict()
    off, p_off = step(), predict()
    with deterministic():
        on2, p2 = step(), predict()
    assert_bit_equal("training step on / off / on", on1, on2)
    assert_bit_equal("rew_end predict on / off / on", p1, p2)
    assert TD._rel(off[0], on1[0]) < 1e-3 and TD._rel(p_off[0], p1[0]) < 1e-3


def test_workspace_queries_in_both_modes():
    """The workspace queries plan in the handle's mode: the default net's inference and training workspaces are the same size
    in both (the colsum partials reuse the wgrad partial buffer); a net whose largest activation is an 8 x 8 attention level
    needs more backward temporaries for the split attention backward in deterministic mode."""
    dev = TD._dev()
    from diamond_b200 import _lib

    lib = _lib.lib()
    sizes = {}
    for name, inner, hw in (("default", O.InnerCfg(), 64),
                            ("attn8", O.InnerCfg(cond_channels=64, depths=[1], channels=[64], attn_depths=[1]), 8)):
        den, _ = TD._build(inner, 3, dev)
        h = den.inner_model._native()
        for on in (0, 1):
            _lib.check(lib.dmd_denoiser_set_deterministic(h, on))
            sizes[name, on] = (lib.dmd_denoiser_workspace_bytes(h, 32, hw, hw), lib.dmd_denoiser_train_workspace_bytes(h, 32, hw, hw))
        _lib.check(lib.dmd_denoiser_set_deterministic(h, 0))
    print(sizes)
    assert all(v > 0 for pair in sizes.values() for v in pair)
    assert sizes["default", 0] == sizes["default", 1]
    assert sizes["attn8", 0][0] == sizes["attn8", 1][0] and sizes["attn8", 1][1] > sizes["attn8", 0][1]
