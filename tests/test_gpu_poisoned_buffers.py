"""Every native entry point on poisoned scratch memory: a kernel that reads a byte no earlier launch of the same call wrote
must change the result.

Each case runs the same calls twice, once on fresh memory and once with every buffer the workspace contract calls scratch
or output (include/diamond_b200.h, "Workspace contract") filled with a byte pattern first -- the package's own allocations
(torch.empty / empty_like inside diamond_b200), the cached inference and backward workspaces, the pooled training workspaces
between optimizer steps, the sampler's trajectory slots >= 1 and the wgrad partial buffers.  Inputs, weights, optimizer state
and a training workspace between its forward and its backward are never poisoned.  The patterns:

* 0x00 -- zeros, what fresh memory often holds, so a missed write can look right;
* 0xFF -- NaN in fp16, fp32 and fp64;
* 0x5A -- large and finite in fp16 (203.25), fp32 (1.5e16) and fp64 (1.5e127): caught where NaN-tolerant code (fmaxf, a
  comparison) would hide a NaN.

The two runs are compared with the criterion the suite uses for two clean runs of the same call: the GroupNorm statistics
accumulate with fp64 atomics, so the last bit of an output may move (DESIGN.md section 2).  Everything must be finite; model
outputs, logits and states agree to 1e-6 relative L2; quantised frames differ in fewer than 1e-3 of their pixels; optimizer
results and lambda-returns are bit-identical.  A training call is run clean twice, and its gradients, losses and updated
parameters may move by twice the largest clean run-to-run difference: the norm backward adds its sums with fp32 atomics, which
moves a gradient by up to ~3e-4 relative L2 between two clean runs of the small nets measured here (NVIDIA H100 80GB HBM3,
700 W).  Zeroed FiLM gradient offsets moved the gradients by 0.14 to 0.18.  A negative control poisons a training workspace
between its forward and its backward, which the contract forbids, and must fail the same check.
"""
import contextlib
import importlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import torch_oracle as O

PATTERNS = [0x00, 0xFF, 0x5A]
BYTES = pytest.mark.parametrize("byte", PATTERNS, ids=lambda b: f"0x{b:02X}")
REL = 1e-6          # relative L2 of two runs of a call that differ only in the order of the fp64 GroupNorm atomics
PIXELS = 1e-3       # share of quantised pixels allowed to move (a value that sits on a quantiser bucket edge)

# the modules that allocate what they hand to the native library
_ALLOCATING_MODULES = ["diamond_b200.utils", "diamond_b200.ops", "diamond_b200.optim", "diamond_b200.models.diffusion.inner_model",
                       "diamond_b200.models.diffusion.denoiser", "diamond_b200.models.diffusion.diffusion_sampler",
                       "diamond_b200.models.rew_end_model", "diamond_b200.models.actor_critic"]


def poison_(t: torch.Tensor, byte: int) -> torch.Tensor:
    """Fills every byte of the contiguous tensor `t` with `byte`."""
    assert t.is_contiguous()
    if t.numel():
        t.reshape(-1).view(torch.uint8).fill_(byte)
    return t


class _PoisonedTorch:
    """`torch` as the package's modules see it inside `poisoned_allocations`: empty / empty_like return CUDA tensors filled
    with the pattern; everything else is torch."""

    def __init__(self, byte):
        self._byte = byte

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *a, **k):
        t = torch.empty(*a, **k)
        return poison_(t, self._byte) if t.is_cuda else t

    def empty_like(self, *a, **k):
        t = torch.empty_like(*a, **k)
        return poison_(t, self._byte) if t.is_cuda and t.is_contiguous() else t


@contextlib.contextmanager
def poisoned_allocations(byte):
    """Every CUDA tensor the package allocates with torch.empty / empty_like comes back filled with `byte` (None: no-op)."""
    if byte is None:
        yield
        return
    mods = [importlib.import_module(m) for m in _ALLOCATING_MODULES]
    proxy = _PoisonedTorch(byte)
    for m in mods:
        assert m.torch is torch
        m.torch = proxy
    try:
        yield
    finally:
        for m in mods:
            m.torch = torch


def poison_scratch(byte, *modules):
    """The scratch the package caches between calls: inference workspaces, pooled training workspaces (not live ones: those are
    held by their autograd node, not the pool), the actor-critic backward scratch and the wgrad partial buffers."""
    if byte is None:
        return
    from diamond_b200 import ops

    for m in modules:
        d = m.__dict__
        for t in [d.get("_ws"), d.get("_bwd_scratch")] + list(d.get("_ws_pool", [])):
            if t is not None:
                poison_(t, byte)
    for t in ops._partial.values():
        poison_(t, byte)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _check_close(label, got, ref, again=None, rel=REL):
    """got / ref: dicts of tensors from the poisoned and the clean run.  again: a second clean run of a call whose backward
    accumulates with fp32 / fp64 atomics (norm backward sums, GroupNorm statistics); every tensor may then move by twice the
    largest clean run-to-run difference of the call (a loss after an optimizer step inherits the gradients' difference)."""
    assert got.keys() == ref.keys()
    bound = rel if again is None else max([rel] + [2 * _rel(again[k], ref[k]) for k in ref])
    worst = 0.0
    for k in ref:
        assert torch.isfinite(ref[k]).all(), f"{label}: clean {k} is not finite"
        assert torch.isfinite(got[k]).all(), f"{label}: {k} is not finite after poisoning"
        e = _rel(got[k], ref[k])
        worst = max(worst, e)
        assert e <= bound, f"{label}: {k} moved by {e:.3e} (relative L2) after poisoning, bound {bound:.3e}"
    print(f"{label}: worst relative L2 difference {worst:.2e}, bound {bound:.2e}")


def _check_pixels(label, got, ref):
    assert torch.isfinite(got).all(), f"{label}: not finite after poisoning"
    frac = float(((got - ref).abs() > 1e-6).float().mean())
    print(f"{label}: {frac:.2e} of the pixels moved")
    assert frac < PIXELS, (label, frac)


def _check_equal(label, got, ref):
    for k in ref:
        assert torch.equal(got[k], ref[k]), f"{label}: {k} is not bit-identical after poisoning"


# ------------------------------------------------------------------------------------------------ helpers
def _inner_cfg(name):
    if name == "default":
        return O.InnerCfg()
    if name == "attn8":       # attention at the 8x8 level of the default net: 121 tokens at 84x84 (88x88 padded)
        return O.InnerCfg(attn_depths=[0, 0, 0, 1])
    from oracle.make_golden import CASES

    return CASES["denoiser_small_heun"]["inner"]   # 3 levels, attention inside the 64-channel level


def _denoiser(name, dev, seed=3):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.synthetic import randomize_module_

    i = _inner_cfg(name)
    den = Denoiser(DenoiserConfig(InnerModelConfig(i.img_channels, i.num_steps_conditioning, i.cond_channels, list(i.depths),
                                                   list(i.channels), list(i.attn_depths), i.num_actions), 0.5, 0.3))
    randomize_module_(den.inner_model, seed)
    den = den.to(dev)
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    return den, i


def _rew_end(dev, seed=4):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import randomize_module_

    c = O.RewEndCfg()
    m = RewEndModel(RewEndModelConfig(c.lstm_dim, c.img_channels, c.img_size, c.cond_channels, list(c.depths), list(c.channels),
                                      list(c.attn_depths), c.num_actions))
    randomize_module_(m, seed)
    return m.to(dev), c


def _levels(shape, seed, dev):
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.integers(0, 256, size=shape, dtype=np.uint8)).to(dev)


# ------------------------------------------------------------------------------------------------ the poison helper (CPU)
def test_poison_writes_the_patterns_it_claims():
    for dt in (torch.float16, torch.float32, torch.float64):
        t = torch.ones(7, 3, dtype=dt)
        assert torch.equal(poison_(t, 0x00), torch.zeros(7, 3, dtype=dt))
        assert torch.isnan(poison_(t, 0xFF)).all()
        v = poison_(t, 0x5A)
        assert torch.isfinite(v).all() and bool((v == v[0, 0]).all())
        assert float(v[0, 0]) > 200, (dt, float(v[0, 0]))
        assert (t.view(torch.uint8) == 0x5A).all()
    assert float(poison_(torch.empty(1, dtype=torch.float16), 0x5A)) == 203.25
    assert float(poison_(torch.empty(1, dtype=torch.float32), 0x5A)) > 1e16
    assert float(poison_(torch.empty(1, dtype=torch.float64), 0x5A)) > 1e127


def test_poisoned_allocations_reach_the_package_only():
    """The proxy poisons what the package allocates and leaves the test's own allocations alone."""
    from diamond_b200 import utils

    with poisoned_allocations(0xFF):
        assert utils.torch is not torch and utils.torch.zeros is torch.zeros
    assert utils.torch is torch


# ------------------------------------------------------------------------------------------------ denoiser inference
DENOISE_CASES = [("default", 1, 64, 64), ("default", 3, 64, 64), ("default", 32, 64, 64), ("default", 2, 60, 62),
                 ("attn8", 2, 84, 84), ("small", 3, 32, 32)]


@pytest.mark.gpu
@BYTES
@pytest.mark.parametrize("net,b,h,w", DENOISE_CASES)
def test_denoise_and_inner_model_on_poisoned_memory(net, b, h, w, byte):
    """Denoiser.denoise and InnerModel.forward (fp32 and uint8 frame stacks), each called twice on the same cached workspace
    with the workspace poisoned before each call."""
    dev = _dev()
    from diamond_b200 import frames as F

    den, i = _denoiser(net, dev)
    den.eval()
    im = den.inner_model
    T, Cc = i.num_steps_conditioning, i.img_channels
    g = torch.Generator().manual_seed(b * 1000 + h)
    lv = _levels((b, T, Cc, h, w), b + h, dev)
    kinds = torch.full((b, T), F.KIND_CPU, dtype=torch.uint8, device=dev)
    obs = F.decode(lv, kinds)
    act = torch.randint(0, i.num_actions, (b, T), generator=g).to(dev)
    noisy = torch.randn(b, Cc, h, w, generator=g).to(dev)
    sigma = torch.rand(b, generator=g).add(0.1).to(dev)
    ctx = F.U8FrameStack(lv, kinds, F.context_table(dev, 0.5))

    def run(p):
        out = {}
        with torch.no_grad():
            for k in range(2):
                poison_scratch(p, im)
                with poisoned_allocations(p):
                    out[f"denoised{k}"] = den.denoise(noisy, sigma, obs.reshape(b, T * Cc, h, w), act)
                    out[f"inner{k}"] = im(noisy * 0.7, sigma.log() / 4, obs.reshape(b, T * Cc, h, w) / 0.5, act)
                    out[f"inner_u8_{k}"] = im(noisy * 0.7, sigma.log() / 4, ctx, act)
        torch.cuda.synchronize()
        return out

    ref = run(None)
    _check_close(f"denoise {net} B={b} {h}x{w} 0x{byte:02X}", run(byte), ref)


# ------------------------------------------------------------------------------------------------ sampler and imagined env
@pytest.mark.gpu
@BYTES
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("kind", ["euler", "heun", "churn"])
def test_sampler_on_poisoned_memory(kind, graph, byte):
    """DiffusionSampler.sample called three times (graph replays): the workspace and trajectory slots >= 1 are poisoned before
    every call."""
    dev = _dev()
    from diamond_b200.models.diffusion import DiffusionSampler, DiffusionSamplerConfig

    net = "small" if kind != "euler" else "default"
    den, i = _denoiser(net, dev)
    den.eval()
    b, hw = 3, 32 if net == "small" else 64
    cfg = {"euler": DiffusionSamplerConfig(3), "heun": DiffusionSamplerConfig(3, order=2),
           "churn": DiffusionSamplerConfig(4, order=2, s_churn=1.0)}[kind]
    lv = _levels((b, i.num_steps_conditioning, i.img_channels, hw, hw), 5, dev)
    prev = lv.float().div(255).mul(2).sub(1)
    act = torch.randint(0, i.num_actions, (b, i.num_steps_conditioning), generator=torch.Generator().manual_seed(6)).to(dev)

    def run(p):
        sampler = DiffusionSampler(den, cfg)
        sampler.use_cuda_graph = graph
        outs = []
        for k in range(3):
            torch.manual_seed(10 + k)
            if p is not None and sampler._buf:
                poison_(next(iter(sampler._buf.values()))["traj"][1:], p)
            poison_scratch(p, den.inner_model)
            with poisoned_allocations(p):
                x, traj = sampler.sample(prev, act)
            outs.append(torch.stack(traj[1:]))
        torch.cuda.synchronize()
        return torch.stack(outs)

    ref = run(None)
    _check_pixels(f"sample {kind} graph={graph} 0x{byte:02X}", run(byte), ref)


@pytest.mark.gpu
@BYTES
def test_world_model_env_on_poisoned_memory(byte):
    """WorldModelEnv over two full cycles of its ring heads (horizon 3 forces deaths and re-initialisations): the denoiser and
    reward/termination workspaces and the trajectory slots >= 1 are poisoned before every step."""
    dev = _dev()
    from diamond_b200.envs.world_model_env import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.diffusion import DiffusionSamplerConfig

    den, i = _denoiser("default", dev)
    den.eval()
    rew_end, _ = _rew_end(dev)
    rew_end.eval()
    for p in rew_end.parameters():
        p.requires_grad_(False)

    class Loader:
        batch_sampler = SimpleNamespace(batch_size=8)

        def __iter__(self):
            rng = np.random.default_rng(0)
            while True:
                levels = torch.from_numpy(rng.integers(0, 256, size=(8, 4, 3, 64, 64), dtype=np.uint8))
                yield SimpleNamespace(obs=levels, act=torch.from_numpy(rng.integers(0, 4, size=(8, 4)).astype(np.int64)))

    def run(p):
        env = WorldModelEnv(den, rew_end, Loader(), WorldModelEnvConfig(3, 2, DiffusionSamplerConfig(3)))
        torch.manual_seed(0)
        with poisoned_allocations(p):
            env.reset()
        out = {"frames": [], "rew": [], "end": [], "trunc": []}
        for step in range(2 * i.num_steps_conditioning):
            a = torch.randint(0, 4, (8,), device=dev)
            if p is not None and env.sampler._buf:
                poison_(next(iter(env.sampler._buf.values()))["traj"][1:], p)
            poison_scratch(p, den.inner_model, rew_end)
            with poisoned_allocations(p):
                obs, rew, end, trunc, _ = env.step(a)
            for k, v in (("frames", obs), ("rew", rew), ("end", end), ("trunc", trunc)):
                out[k].append(v.clone())
        out["ring"] = [env._frames.clone()]
        torch.cuda.synchronize()
        return {k: torch.stack(v) for k, v in out.items()}

    ref = run(None)
    got = run(byte)
    assert int(ref["end"].sum() + ref["trunc"].sum()) >= 8, "the horizon must force deaths"
    _check_pixels(f"WorldModelEnv frames 0x{byte:02X}", got["frames"], ref["frames"])
    _check_pixels(f"WorldModelEnv ring 0x{byte:02X}", got["ring"], ref["ring"])
    for k in ("rew", "end", "trunc"):
        assert torch.equal(got[k], ref[k]), k


# ------------------------------------------------------------------------------------------------ denoiser training
class _Batch:
    def __init__(self, obs, act, mask):
        self.obs, self.act, self.mask_padding = obs, act, mask


def _denoiser_training(net, byte, dev, steps=2, poison_live=None):
    """Two optimizer steps (clip_grad_norm_ + AdamW), each over Denoiser.forward with two autoregressive steps + backward.
    The pooled training workspaces are poisoned between the optimizer steps.  poison_live: also poison every live training
    workspace between its forward and its backward (the negative control)."""
    from diamond_b200 import optim

    den, i = _denoiser(net, dev)
    den.train()
    im = den.inner_model
    b, hw = (4, 64) if net == "default" else (3, 32)
    T = i.num_steps_conditioning + 2
    obs = _levels((b, T, i.img_channels, hw, hw), 7, dev).float().div(255).mul(2).sub(1)
    act = torch.randint(0, i.num_actions, (b, T), generator=torch.Generator().manual_seed(8)).to(dev)
    batch = _Batch(obs, act, torch.ones(b, T, dtype=torch.bool, device=dev))
    opt = optim.AdamW(den.parameters(), lr=1e-3)
    live = []
    if poison_live is not None:
        acquire = im._acquire_ws
        im._acquire_ws = lambda n: live.append(acquire(n)) or live[-1]
    out = {}
    for s in range(steps):
        poison_scratch(byte, im)
        torch.manual_seed(100 + s)
        with poisoned_allocations(byte):
            opt.zero_grad(set_to_none=True)
            loss, _ = den(batch)
            for ws in live:
                poison_(ws, poison_live)
            live.clear()
            loss.backward()
            out[f"loss{s}"] = loss.detach().reshape(1)
            out[f"grad{s}"] = torch.cat([p.grad.reshape(-1) for p in den.parameters()])
            optim.clip_grad_norm_(den.parameters(), 1.0)
            opt.step()
        out[f"param{s}"] = torch.cat([p.detach().reshape(-1) for p in den.parameters()])
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@BYTES
@pytest.mark.parametrize("net", ["default", "small"])
def test_denoiser_training_on_poisoned_memory(net, byte):
    """The flat gradient buffers, the outputs and the reused training workspaces start poisoned.  A training workspace only
    has to keep its contents from a forward to its backward: state the backward needs across optimizer steps (the FiLM
    gradient offsets) lives with the model."""
    dev = _dev()
    ref, again = _denoiser_training(net, None, dev), _denoiser_training(net, None, dev)
    _check_close(f"denoiser training {net} 0x{byte:02X}", _denoiser_training(net, byte, dev), ref, again)


@pytest.mark.gpu
@BYTES
def test_poisoning_a_live_training_workspace_is_seen(byte):
    """Negative control: poisoning the training workspaces between their forward and their backward (which the contract
    forbids) gives non-finite or visibly moved gradients, so the harness does see reads of poisoned memory."""
    dev = _dev()
    ref = _denoiser_training("small", None, dev, steps=1)
    bad = _denoiser_training("small", None, dev, steps=1, poison_live=byte)
    g, r = bad["grad0"], ref["grad0"]
    finite = bool(torch.isfinite(g).all())
    e = _rel(g, r) if finite else float("inf")
    print(f"live workspace poisoned with 0x{byte:02X}: gradients finite {finite}, relative L2 difference {e:.3e}")
    assert not finite or e > 1e3 * REL


@pytest.mark.gpu
def test_training_workspace_reused_through_the_c_abi():
    """dmd_inner_model_forward_train + dmd_denoiser_backward on one workspace through ctypes, same inputs every call: twice on an
    untouched workspace (the clean run-to-run difference), then with the workspace poisoned between a backward and the next
    forward, and with poisoned outputs and gradient buffers.  Before the FiLM gradient offsets moved into the packed weights,
    a zeroed workspace sent every FiLM weight gradient to flat elements [0, cond_channels)."""
    dev = _dev()
    from diamond_b200 import _lib

    lib = _lib.lib()
    den, i = _denoiser("small", dev)
    im = den.inner_model
    h = im.native()
    b, hw, T, Cc = 3, 32, i.num_steps_conditioning, i.img_channels
    g = torch.Generator().manual_seed(9)
    noisy = torch.randn(b, Cc, hw, hw, generator=g).to(dev)
    cn = torch.randn(b, generator=g).to(dev)
    obs = torch.randn(b, T * Cc, hw, hw, generator=g).to(dev)
    act = torch.randint(0, i.num_actions, (b, T), generator=g).to(dev)
    gout = torch.randn(b, Cc, hw, hw, generator=g).to(dev)
    ws = poison_(torch.empty(lib.dmd_denoiser_train_workspace_bytes(h, b, hw, hw), dtype=torch.uint8, device=dev), 0x5A)
    _, _, total = im.grad_layout()
    runs = []
    for byte in (None, None, 0x00, 0xFF, 0x5A):
        if byte is not None:
            poison_(ws, byte)
        out = poison_(torch.empty_like(noisy), 0xFF if byte is None else byte)
        grads = poison_(torch.empty(total, device=dev), 0xFF if byte is None else byte)
        st = _lib.current_stream()
        _lib.check(lib.dmd_inner_model_forward_train(h, b, hw, hw, noisy.data_ptr(), cn.data_ptr(), 0, obs.data_ptr(), act.data_ptr(),
                                                     out.data_ptr(), ws.data_ptr(), ws.numel(), st))
        _lib.check(lib.dmd_denoiser_backward(h, b, hw, hw, gout.data_ptr(), grads.data_ptr(), total, ws.data_ptr(), st))
        torch.cuda.synchronize()
        runs.append({"out": out.clone(), "grads": grads.clone()})
    ref, again = runs[0], {"out": runs[0]["out"], "grads": runs[1]["grads"]}   # the forward is deterministic here
    assert torch.equal(runs[1]["out"], ref["out"])
    for k, r in enumerate(runs[2:]):
        _check_close(f"C ABI training call {k + 3}", r, ref, again)


# ------------------------------------------------------------------------------------------------ reward / termination model
def _rew_end_inputs(dev, b=32, t=19):
    from diamond_b200 import frames as F

    lv, nlv = _levels((b, t, 3, 64, 64), 11, dev), _levels((b, t, 3, 64, 64), 12, dev)
    kinds = torch.full((b, t), F.KIND_CPU, dtype=torch.uint8, device=dev)
    kinds[::5, t // 2:] = F.KIND_PADDING
    act = torch.randint(0, 4, (b, t), generator=torch.Generator().manual_seed(13)).to(dev)
    return lv, nlv, kinds, act


@pytest.mark.gpu
@BYTES
def test_rew_end_predict_on_poisoned_memory(byte):
    """predict_rew_end at 32 x 19, from fp32 and uint8 frames, with and without a carried state; the cached workspace is
    poisoned before every call."""
    dev = _dev()
    from diamond_b200 import frames as F

    m, _ = _rew_end(dev)
    m.eval()
    for p in m.parameters():
        p.requires_grad_(False)
    lv, nlv, kinds, act = _rew_end_inputs(dev)
    obs, nobs = F.decode(lv, kinds), F.decode(nlv, kinds)

    def run(p):
        out = {}
        state = None
        for k, u8 in enumerate((False, True, False)):
            poison_scratch(p, m)
            with torch.no_grad(), poisoned_allocations(p):
                if u8:
                    r, e, state = m.predict_rew_end(lv, act, nlv, state, kinds=(kinds, kinds))
                else:
                    r, e, state = m.predict_rew_end(obs, act, nobs, state)
            out.update({f"rew{k}": r, f"end{k}": e, f"hx{k}": state[0], f"cx{k}": state[1]})
        torch.cuda.synchronize()
        return out

    ref = run(None)
    _check_close(f"rew_end predict 0x{byte:02X}", run(byte), ref)


@pytest.mark.gpu
@BYTES
def test_rew_end_training_on_poisoned_memory(byte):
    """RewEndModel.forward + backward at 32 x 19, two optimizer steps; pooled workspaces poisoned between the steps."""
    dev = _dev()
    from diamond_b200 import optim
    from test_gpu_rew_end_training import _batch, _seeded_batch

    obs, act, rew, end, mask, final_obs = _seeded_batch(32, 19, 2024)

    def run(p):
        m, _ = _rew_end(dev)
        m.train()
        batch = _batch(obs, act, rew, end, mask, final_obs, dev)
        opt = optim.AdamW(m.parameters(), lr=1e-4)
        out = {}
        for s in range(2):
            poison_scratch(p, m)
            with poisoned_allocations(p):
                opt.zero_grad(set_to_none=True)
                loss, _ = m(batch)
                loss.backward()
                out[f"loss{s}"] = loss.detach().reshape(1)
                out[f"grad{s}"] = torch.cat([q.grad.reshape(-1) for q in m.parameters()])
                optim.clip_grad_norm_(m.parameters(), 10.0)
                opt.step()
            out[f"param{s}"] = torch.cat([q.detach().reshape(-1) for q in m.parameters()])
        torch.cuda.synchronize()
        return out

    ref, again = run(None), run(None)
    _check_close(f"rew_end training 0x{byte:02X}", run(byte), ref, again)


# ------------------------------------------------------------------------------------------------ actor-critic
@pytest.mark.gpu
@BYTES
def test_actor_critic_update_on_poisoned_memory(byte, monkeypatch):
    """Two actor-critic updates over 32 envs x 15 steps with deaths and burn-in (forward, backward and the accumulated
    backward of every node); workspaces, pooled workspaces and the backward scratch are poisoned between the updates."""
    dev = _dev()
    from test_gpu_imagination_models import AC_SEED, AC_T, _bench_rollout_data, _native_ac, _run_native_updates

    d = _bench_rollout_data()

    def run(p):
        ac = _native_ac(O.seeded_actor_critic_state_dict(O.ActorCriticCfg(), AC_SEED), dev)
        out = {}
        for u in range(2):
            ac.env_loop = ac.loss_cfg = None   # a fresh rollout of the scripted env per update
            poison_scratch(p, ac)
            with poisoned_allocations(p):
                r = _run_native_updates(ac, d, AC_T, 1, monkeypatch, dev)[0]
            out.update({f"loss{u}": torch.tensor([r["loss"]]), f"logits{u}": r["logits"], f"val{u}": r["val"],
                        f"grad{u}": torch.cat([g.reshape(-1) for g in r["grads"].values()])})
        return out

    ref, again = run(None), run(None)
    _check_close(f"actor-critic 0x{byte:02X}", run(byte), ref, again)


@pytest.mark.gpu
@BYTES
def test_lambda_returns_on_poisoned_memory(byte):
    dev = _dev()
    from diamond_b200.models.actor_critic import compute_lambda_returns

    g = torch.Generator().manual_seed(1)
    rew, vb = torch.randn(32, 15, generator=g).to(dev), torch.randn(32, 15, generator=g).to(dev)
    end = (torch.rand(32, 15, generator=g) < 0.1).long().to(dev)
    trunc = (torch.rand(32, 15, generator=g) < 0.1).long().to(dev)
    ref = compute_lambda_returns(rew, end, trunc, vb, 0.985, 0.95)
    with poisoned_allocations(byte):
        got = compute_lambda_returns(rew, end, trunc, vb, 0.985, 0.95)
    _check_equal(f"lambda-returns 0x{byte:02X}", {"r": got}, {"r": ref})


# ------------------------------------------------------------------------------------------------ optimizer
@pytest.mark.gpu
@BYTES
def test_clip_and_adamw_on_poisoned_memory(byte):
    """clip_grad_norm_ + AdamW.step three times over the denoiser's parameters with fixed gradients: the norm's partial
    buffer (allocated per call) comes back poisoned.  Results are bit-identical: the reduction has a fixed order."""
    dev = _dev()
    from diamond_b200 import optim

    def run(p):
        den, _ = _denoiser("default", dev)
        params = list(den.parameters())
        g = torch.Generator().manual_seed(21)
        for q in params:
            q.grad = torch.randn(q.shape, generator=g).mul(0.01).to(dev)
        opt = optim.AdamW(params, lr=1e-3, weight_decay=0.01)
        out = {}
        for s in range(3):
            with poisoned_allocations(p):
                out[f"norm{s}"] = optim.clip_grad_norm_(params, 0.5).reshape(1)
                opt.step()
            out[f"param{s}"] = torch.cat([q.detach().reshape(-1) for q in params])
            out[f"grad{s}"] = torch.cat([q.grad.reshape(-1) for q in params])
        torch.cuda.synchronize()
        return out

    ref = run(None)
    got = run(byte)
    assert all(torch.isfinite(v).all() for v in got.values())
    _check_equal(f"clip + AdamW 0x{byte:02X}", got, ref)
