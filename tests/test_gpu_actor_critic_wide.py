"""GPU: actor-critics with 128-channel levels (WIDE_AC_CASES of oracle/make_golden_wide_actor_critic.py: [64, 128, 128, 128],
[128] * 4 and [32, 128, 64, 128]).  Their 3x3 128 -> 128 convs run split-fp16 as three passes per 64-channel K chunk, their
dgrad in 64-channel gradient chunks and their weight gradients in 64 x 64 blocks.

- create takes every mix of 32, 64 and 128 over four levels;
- the forward at B = 1, 5 and 32 against the reference's outputs (tests/golden/actor_critic_wide.npz), 1e-3 relative L2;
- one backward node (the case's levels at 8 x 8 without max-pools) against float64 autograd, with the bounds of the
  fp16-operand emulation (oracle/fp16_emulation.py grad_errors, as tests/test_gpu_training_configs.py): whole gradient
  within 1.25x the emulation's error, each tensor (parameters, hx_in, cx_in) within 2x its own or negligible;
- backward_accumulate over two nodes equals the sum of two backward calls, to fp32 rounding;
- torch.autograd.grad (accumulate_native_grads = False) equals the adopted .grad;
- the imagination update (32 envs x horizon 15, dead-env burn-in, a second update carrying the detached state) of the
  [64, 128, 128, 128] policy against the float64 oracle;
- NaN-filled workspace, scratch and outputs give the results of clean buffers;
- the default [32, 32, 64, 64] policy launches as many kernels per forward and per backward as before 128-channel levels."""
import dataclasses
import itertools
import math
import os

import numpy as np
import pytest
import torch
from torch.distributions.categorical import Categorical

from diamond_b200 import _lib
from oracle import fp16_emulation as E
from oracle import torch_oracle as O
from oracle.make_golden import frames_from_u8
from oracle.make_golden_wide_actor_critic import FWD_STEPS, WIDE_AC_CASES, wide_ac_inputs

gpu = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "actor_critic_wide.npz")
FWD_TOL = 1e-3
WHOLE_MARGIN, TENSOR_MARGIN = 1.25, 2.0     # tests/test_gpu_training_configs.py
LOGITS_TOL, VAL_TOL, GRAD_TOL, TENSOR_TOL, PER_TENSOR_CAP = 1e-3, 2e-3, 1e-3, 4e-3, 5e-3   # tests/test_gpu_imagination_models.py
# kernel launches of the default [32, 32, 64, 64] policy (lstm_dim 512, 64 x 64 frames) at B = 32, counted with
# dmd_launch_count on the commit before 128-channel actor-critic levels
DEFAULT_FWD_LAUNCHES = 24
DEFAULT_BWD_LAUNCHES = 64
# accumulate_native_grads = False against the adopted .grad: they differ in the order of fp32 additions across nodes and in
# the fp64 atomics of the GroupNorm sums, which also make two identical backward calls differ.  Measured on an H100 80GB
# HBM3 (700 W): 1.24e-6 whole and 1.16e-5 in one tensor (encoder.encoder.0.weight) for [128] * 4
AUTOGRAD_WHOLE_TOL, AUTOGRAD_TENSOR_TOL = 5e-6, 5e-5
F64 = torch.float64


@pytest.fixture
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden():
    g = np.load(GOLDEN)
    return {name: {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")} for name in WIDE_AC_CASES}


def _threads():
    torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _native_ac(cfg, sd, dev):
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig

    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    ac.load_state_dict(sd)
    return ac.to(dev).train()


def _case_ac(name, dev):
    c = WIDE_AC_CASES[name]
    return _native_ac(c["cfg"], O.seeded_actor_critic_state_dict(c["cfg"], c["wseed"]), dev)


def _config(channels):
    c = _lib.ActorCriticConfigC(lstm_dim=512, img_channels=3, img_size=64, num_levels=len(channels), num_actions=4)
    for i, ch in enumerate(channels):
        c.channels[i], c.down[i] = ch, 1
    return c


# ------------------------------------------------------------------------------------------------ create
@gpu
def test_create_accepts_every_mix(dev):
    lib = _lib.lib()
    for channels in itertools.product([32, 64, 128], repeat=4):
        h = lib.dmd_actor_critic_create(_config(list(channels)))
        assert h, (channels, lib.dmd_last_error().decode())
        assert lib.dmd_actor_critic_workspace_bytes(h, 32) > 0 and lib.dmd_actor_critic_backward_scratch_bytes(h, 32) > 0
        lib.dmd_actor_critic_destroy(h)


# ------------------------------------------------------------------------------------------------ forward
@gpu
@pytest.mark.parametrize("name", list(WIDE_AC_CASES))
@pytest.mark.parametrize("b", [1, 5, 32])
def test_forward_matches_reference(dev, golden, name, b):
    g = golden[name]
    ac = _case_ac(name, dev)
    x = wide_ac_inputs(name)
    hx, cx = x["hx0"][:b].to(dev), x["cx0"][:b].to(dev)
    errs = []
    with torch.no_grad():
        for t in range(FWD_STEPS):
            logits, val, (hx, cx) = ac.predict_act_value(x["fwd_obs"][t, :b].to(dev), (hx, cx))
            errs += [_rel(logits, torch.from_numpy(g["fwd_logits"][t, :b])), _rel(val, torch.from_numpy(g["fwd_val"][t, :b]))]
    errs += [_rel(hx, torch.from_numpy(g["fwd_hx"][:b])), _rel(cx, torch.from_numpy(g["fwd_cx"][:b]))]
    print(f"{name} B={b}: worst relative L2 {max(errs):.2e} (logits / value per step, hx, cx)")
    assert max(errs) < FWD_TOL, errs


# ------------------------------------------------------------------------------------------------ one backward node
NODE_B = 8


def _node_cfg(cfg):
    """The case's levels at 8 x 8 frames without max-pools, as the actor-critic cases of tests/test_gpu_training_configs.py:
    the emulation runs the forward in float64, and a max-pool window whose two largest inputs differ by less than the fp32
    forward's rounding picks another arg-max there, an error the emulation does not model (measured on an H100 80GB HBM3 at
    700 W, [32, 128, 64, 128] at 64 x 64 with max-pools: 1.36x the emulated whole-gradient error, every tensor within 2x its
    own).  The K-split convs, dgrad chunks and weight-gradient blocks depend on the channels only."""
    return dataclasses.replace(cfg, img_size=8, down=[0] * len(cfg.channels))


def _node_inputs(cfg, seed=5):
    gen = torch.Generator().manual_seed(seed)
    obs = torch.rand(NODE_B, cfg.img_channels, cfg.img_size, cfg.img_size, generator=gen) * 2 - 1
    hx = torch.randn(NODE_B, cfg.lstm_dim, generator=gen) * 0.3
    cx = torch.randn(NODE_B, cfg.lstm_dim, generator=gen) * 0.3
    # the loss: a fixed random linear functional of every output
    w = [torch.randn(NODE_B, cfg.num_actions, generator=gen), torch.randn(NODE_B, generator=gen),
         torch.randn(NODE_B, cfg.lstm_dim, generator=gen), torch.randn(NODE_B, cfg.lstm_dim, generator=gen)]
    return obs, hx, cx, w


def _node_loss(outs, w):
    return sum((o * wi.to(o)).sum() for o, wi in zip(outs, w))


@gpu
@pytest.mark.parametrize("name", list(WIDE_AC_CASES))
def test_backward_node_matches_float64(dev, name):
    c = WIDE_AC_CASES[name]
    cfg = _node_cfg(c["cfg"])
    obs, hx, cx, w = _node_inputs(cfg)
    ac = _native_ac(cfg, O.seeded_actor_critic_state_dict(cfg, c["wseed"]), dev)
    hx_d, cx_d = hx.to(dev).requires_grad_(True), cx.to(dev).requires_grad_(True)
    logits, val, (ho, co) = ac.predict_act_value(obs.to(dev), (hx_d, cx_d))
    _node_loss([logits, val, ho, co], w).backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu() for k, p in ac.named_parameters()}
    grads["hx_in"], grads["cx_in"] = hx_d.grad.cpu(), cx_d.grad.cpu()

    _threads()
    sd = {k: v.to(F64).requires_grad_(True) for k, v in O.seeded_actor_critic_state_dict(cfg, c["wseed"]).items()}
    sd["hx_in"], sd["cx_in"] = hx.to(F64).requires_grad_(True), cx.to(F64).requires_grad_(True)
    obs64 = obs.to(F64)

    def loss_fn(p):
        lg, v, (h2, c2) = O.predict_act_value(obs64, p["hx_in"], p["cx_in"], p, cfg)
        return _node_loss([lg, v, h2, c2], w)
    _, _, emu_whole, emu_per, ref = E.grad_errors(loss_fn, sd, E.actor_critic_stream(sd))
    num = sum(float((grads[k].double() - r).pow(2).sum()) for k, r in ref.items())
    total = math.sqrt(sum(float(r.pow(2).sum()) for r in ref.values()))
    whole = math.sqrt(num) / total
    rows = sorted(((float((grads[k].double() - r).norm() / r.norm().clamp_min(1e-30)), k, float(r.norm())) for k, r in ref.items()), reverse=True)
    print(f"{name}: whole gradient {whole:.3e} (emulation {emu_whole:.3e}, bound {WHOLE_MARGIN * emu_whole:.3e}); "
          f"hx_in {dict((k, e) for e, k, _ in rows)['hx_in']:.2e}, cx_in {dict((k, e) for e, k, _ in rows)['cx_in']:.2e}")
    for e, k, n in rows[:5]:
        print(f"   {e:9.3e}  bound {TENSOR_MARGIN * emu_per[k]:9.3e}  |g|={n:9.3e}  {k}")
    assert whole < WHOLE_MARGIN * emu_whole, (whole, emu_whole)
    for e, k, n in rows:
        assert e <= TENSOR_MARGIN * emu_per[k] or e * n < 1e-4 * total, (k, e, emu_per[k], n, total)
        assert e < PER_TENSOR_CAP, (k, e)


# ------------------------------------------------------------------------------------------------ the C ABI: accumulate, poison
class _Node:
    """One forward through dmd_actor_critic_forward into its own workspace, and its backward through the C ABI."""

    def __init__(self, ac, obs, hx, cx, fill=None):
        lib, dev = _lib.lib(), obs.device
        self.ac, self.h, self.b = ac, ac._native(), obs.size(0)
        self.hx, self.cx = hx.contiguous(), cx.contiguous()
        self.ws = torch.empty(lib.dmd_actor_critic_workspace_bytes(self.h, self.b), dtype=torch.uint8, device=dev)
        self.scratch = torch.empty(lib.dmd_actor_critic_backward_scratch_bytes(self.h, self.b), dtype=torch.uint8, device=dev)
        self.out = [torch.empty(self.b, ac.cfg.num_actions, device=dev), torch.empty(self.b, device=dev),
                    torch.empty_like(self.hx), torch.empty_like(self.cx)]
        self.g_in = [torch.empty_like(self.hx), torch.empty_like(self.cx)]
        for t in [self.ws, self.scratch] + self.out + self.g_in:
            t.view(torch.uint8).fill_(0 if fill is None else fill)
        _lib.check(lib.dmd_actor_critic_forward(self.h, self.b, obs.data_ptr(), self.hx.data_ptr(), self.cx.data_ptr(),
                                                *[o.data_ptr() for o in self.out], self.ws.data_ptr(), self.ws.numel(), _lib.current_stream()))

    def backward(self, g_out, flat, accumulate=False):
        lib = _lib.lib()
        fn = lib.dmd_actor_critic_backward_accumulate if accumulate else lib.dmd_actor_critic_backward
        _lib.check(fn(self.h, self.b, self.hx.data_ptr(), self.cx.data_ptr(), self.out[2].data_ptr(), *[g.data_ptr() for g in g_out],
                      flat.data_ptr(), flat.numel(), self.g_in[0].data_ptr(), self.g_in[1].data_ptr(), self.ws.data_ptr(),
                      self.scratch.data_ptr(), self.scratch.numel(), _lib.current_stream()))


def _node_args(cfg, dev, b, seed):
    gen = torch.Generator().manual_seed(seed)
    obs = (torch.rand(b, cfg.img_channels, cfg.img_size, cfg.img_size, generator=gen) * 2 - 1).to(dev)
    hx, cx = (torch.randn(b, cfg.lstm_dim, generator=gen) * 0.3).to(dev), (torch.randn(b, cfg.lstm_dim, generator=gen) * 0.3).to(dev)
    g_out = [torch.randn(b, cfg.num_actions, generator=gen).to(dev), torch.randn(b, generator=gen).to(dev),
             torch.randn(b, cfg.lstm_dim, generator=gen).to(dev), torch.randn(b, cfg.lstm_dim, generator=gen).to(dev)]
    return obs, hx, cx, g_out


@gpu
@pytest.mark.parametrize("name", list(WIDE_AC_CASES))
def test_backward_accumulate_equals_sum_of_backwards(dev, name):
    cfg = WIDE_AC_CASES[name]["cfg"]
    ac = _case_ac(name, dev)
    total = ac._grad_views_layout()[2]
    a1, a2 = _node_args(cfg, dev, 32, 1), _node_args(cfg, dev, 7, 2)
    n1, n2 = _Node(ac, *a1[:3]), _Node(ac, *a2[:3])
    f1, f2, f12 = (torch.empty(total, device=dev) for _ in range(3))
    n1.backward(a1[3], f1)
    n2.backward(a2[3], f2)
    n1.backward(a1[3], f12)
    n2.backward(a2[3], f12, accumulate=True)
    torch.cuda.synchronize()
    ref = f1.double() + f2.double()
    err = float((f12.double() - ref).norm() / ref.norm())
    print(f"{name}: backward_accumulate vs the sum of two backwards: {err:.2e}")
    assert torch.isfinite(f12).all() and err < 1e-6, err


@gpu
@pytest.mark.parametrize("name", list(WIDE_AC_CASES))
def test_nan_filled_buffers_give_clean_results(dev, name):
    cfg = WIDE_AC_CASES[name]["cfg"]
    ac = _case_ac(name, dev)
    total = ac._grad_views_layout()[2]
    obs, hx, cx, g_out = _node_args(cfg, dev, 32, 3)
    runs = []
    for fill in (None, 0xFF):   # 0xFFFFFFFF is a NaN in fp32 and fp64
        n = _Node(ac, obs, hx, cx, fill)
        flat = torch.empty(total, device=dev)
        flat.view(torch.uint8).fill_(0 if fill is None else fill)
        n.backward(g_out, flat)
        torch.cuda.synchronize()
        runs.append([t.clone() for t in n.out + n.g_in] + [flat])
    for i, (clean, poisoned) in enumerate(zip(*runs)):
        assert torch.isfinite(poisoned).all(), i
        if i < 4:   # the forward has no atomics: bit for bit
            assert torch.equal(clean, poisoned), i
        else:       # the backward's fp32 / fp64 atomic sums may add in another order
            assert _rel(poisoned, clean) < 1e-5, (i, _rel(poisoned, clean))


# ------------------------------------------------------------------------------------------------ autograd surface
class _ScriptedEnv:
    """Pre-generated observations, rewards and flags (the action is ignored); with every death it returns
    `final_observation` and, like WorldModelEnv.step, `burnin_obs` (k, 3, C, H, W) for the k dead envs."""

    def __init__(self, d, dev):
        self.obs_seq, self.rew = d["obs_seq"].to(dev), d["rew"].to(dev)
        self.end_cpu, self.trunc_cpu = d["end"], d["trunc"]
        self.end, self.trunc = d["end"].to(dev), d["trunc"].to(dev)
        self.final_obs = {t: v.to(dev) for t, v in d["final_obs"].items()}
        self.burnin_obs = {t: v.to(dev) for t, v in d["burnin_obs"].items()}
        self.num_envs, self.num_actions, self.t = self.obs_seq.size(1), 4, 0

    def reset(self, seed=None):
        self.t = 0
        return self.obs_seq[0], {}

    def step(self, act):
        t = self.t
        info = {}
        if bool(torch.logical_or(self.end_cpu[t].bool(), self.trunc_cpu[t].bool()).any()):
            info = {"final_observation": self.final_obs[t], "burnin_obs": self.burnin_obs[t]}
        self.t += 1
        return self.obs_seq[t + 1], self.rew[t], self.end[t], self.trunc[t], info


def _run_updates(ac, d, T, n_updates, monkeypatch, dev, accumulate=True):
    """n_updates calls of ActorCritic.forward() on the scripted env, actions replayed, each followed by loss.backward() into
    .grad or by torch.autograd.grad.  Returns per update: loss, logs, logits, values and the gradients by name."""
    from diamond_b200.models.actor_critic import ActorCriticLossConfig

    lc = O.ActorCriticLossCfg(backup_every=T)
    ac.setup_training(_ScriptedEnv(d, dev), ActorCriticLossConfig(lc.backup_every, lc.gamma, lc.lambda_, lc.weight_value_loss,
                                                                  lc.weight_entropy_loss))
    ac.accumulate_native_grads = accumulate
    loop, captured, step = ac.env_loop, [], [0]
    acts = d["act"].to(dev)

    class _Tap:
        def send(self, n):
            captured.append(loop.send(n))
            return captured[-1]

    def replay_sample(self, sample_shape=torch.Size()):
        step[0] += 1
        return acts[:, step[0] - 1]

    ac.env_loop = _Tap()
    monkeypatch.setattr(Categorical, "sample", replay_sample)
    names = [k for k, _ in ac.named_parameters()]
    out = []
    for _ in range(n_updates):
        loss, logs = ac()
        if accumulate:
            loss.backward()
            grads = {k: p.grad.detach().cpu() for k, p in ac.named_parameters()}
            ac.zero_grad(set_to_none=True)
        else:
            gs = torch.autograd.grad(loss, [p for _, p in ac.named_parameters()])
            assert all(p.grad is None for p in ac.parameters())
            grads = {k: g.detach().cpu() for k, g in zip(names, gs)}
        torch.cuda.synchronize()
        out.append(dict(loss=float(loss.detach()), logs={k: float(v) for k, v in logs.items()}, logits=captured[-1][5].detach().cpu(),
                        val=captured[-1][6].detach().cpu(), grads=grads))
    monkeypatch.undo()
    assert step[0] == n_updates * T
    return out


# 32 envs, horizon 15, two updates; deaths per step, each returning 3 burn-in frames (nodes of 1 to 32 rows)
IM_B, IM_T, IM_SEED = 32, 15, 614
IM_DEATHS = {0: [5], 3: [1, 9, 30], 7: [0, 8, 12, 19, 27, 31], 14: list(range(IM_B)), 18: [11, 20], 26: [4, 10, 16]}


def _rollout_data(steps, b, deaths, seed):
    rng = np.random.default_rng(seed)
    img = (3, 64, 64)
    end, trunc = torch.zeros(steps, b, dtype=torch.long), torch.zeros(steps, b, dtype=torch.long)
    final_obs, burnin_obs = {}, {}
    for t, envs in deaths.items():
        for e in envs:
            (trunc if t == IM_T - 1 or (t + e) % 3 == 0 else end)[t, e] = 1
        final_obs[t] = frames_from_u8(rng.integers(0, 256, size=(len(envs),) + img, dtype=np.uint8))
        burnin_obs[t] = frames_from_u8(rng.integers(0, 256, size=(len(envs), 3) + img, dtype=np.uint8))
    return dict(obs_seq=frames_from_u8(rng.integers(0, 256, size=(steps + 1, b) + img, dtype=np.uint8)),
                rew=torch.from_numpy(rng.choice([-1.0, 0.0, 0.0, 2.0], size=(steps, b)).astype(np.float32)), end=end, trunc=trunc,
                final_obs=final_obs, burnin_obs=burnin_obs, act=torch.from_numpy(rng.integers(0, 4, size=(b, steps))))


def _shift(dct, t0, T, dtype):
    return {t - t0: v.to(dtype) for t, v in dct.items() if t0 <= t < t0 + T}


def _oracle_update(cfg, d, sd, t0, T, state=None):
    sl = slice(t0, t0 + T)
    hx, cx = state if state is not None else (None, None)
    logits, val, vb, (hx, cx) = O.actor_critic_rollout(
        d["obs_seq"][t0:t0 + T + 1].to(F64), d["end"][sl], d["trunc"][sl], _shift(d["final_obs"], t0, T, F64), sd, cfg, hx, cx,
        burnin_obs=_shift(d["burnin_obs"], t0, T, F64), return_state=True)
    loss, metrics = O.actor_critic_loss(logits, val, d["act"][:, sl], d["rew"][sl].t().to(F64), d["end"][sl].t().to(F64),
                                        d["trunc"][sl].t().to(F64), vb, O.ActorCriticLossCfg(backup_every=T))
    gs = torch.autograd.grad(loss, list(sd.values()))
    return dict(loss=float(loss.detach()), logs={k: float(v) for k, v in metrics.items()}, logits=logits.detach(), val=val.detach(),
                grads=dict(zip(sd, gs)), state=(hx.detach(), cx.detach()))


def _grad_errors(grads, ref):
    num = den = 0.0
    rows = []
    for k, r in ref.items():
        r = r.double()
        dlt = grads[k].double() - r
        num += float(dlt.pow(2).sum()); den += float(r.pow(2).sum())
        rows.append((float(dlt.norm() / r.norm().clamp_min(1e-30)), k, float(r.norm())))
    return (num / den) ** 0.5, den ** 0.5, sorted(rows, reverse=True)


def _check_update(label, nat, ref):
    T = ref["logits"].size(1)
    e_log = max(_rel(nat["logits"][:, t], ref["logits"][:, t]) for t in range(T))
    e_val = max(_rel(nat["val"][:, t], ref["val"][:, t]) for t in range(T))
    whole, total, rows = _grad_errors(nat["grads"], ref["grads"])
    print(f"{label}: worst logits {e_log:.2e}, values {e_val:.2e}, loss native {nat['loss']:.6f} oracle {ref['loss']:.6f}, "
          f"whole gradient {whole:.2e}; worst tensors " + ", ".join(f"{k} {e:.2e}" for e, k, _ in rows[:4]))
    assert e_log < LOGITS_TOL and e_val < VAL_TOL, (e_log, e_val)
    assert abs(nat["loss"] - ref["loss"]) <= 2e-3 * abs(ref["loss"]) + 1e-5, (nat["loss"], ref["loss"])
    for k, v in ref["logs"].items():
        assert abs(nat["logs"][k] - v) <= 3e-3 * abs(v) + 1e-5, (k, nat["logs"][k], v)
    assert whole < GRAD_TOL, whole
    for e, k, n in rows:
        assert e < TENSOR_TOL or e * n < 1e-4 * total, (k, e, n, total)
        assert e < PER_TENSOR_CAP, (k, e)


@gpu
def test_imagination_update_with_burnin_and_carry_matches_float64(dev, monkeypatch):
    name = "w64_128"
    c = WIDE_AC_CASES[name]
    cfg = c["cfg"]
    d = _rollout_data(2 * IM_T, IM_B, IM_DEATHS, IM_SEED)
    nat = _run_updates(_case_ac(name, dev), d, IM_T, 2, monkeypatch, dev)
    _threads()
    sd = {k: v.to(F64).requires_grad_(True) for k, v in O.seeded_actor_critic_state_dict(cfg, c["wseed"]).items()}
    ref1 = _oracle_update(cfg, d, sd, 0, IM_T)
    _check_update(f"{name} update 1", nat[0], ref1)
    _check_update(f"{name} update 2 (carried state)", nat[1], _oracle_update(cfg, d, sd, IM_T, IM_T, state=ref1["state"]))


@gpu
@pytest.mark.parametrize("name", list(WIDE_AC_CASES))
def test_autograd_grad_equals_adopted_grad(dev, name, monkeypatch):
    d = _rollout_data(5, 6, {1: [2], 3: [0, 4]}, 615)
    acc = _run_updates(_case_ac(name, dev), d, 5, 1, monkeypatch, dev, accumulate=True)[0]
    free = _run_updates(_case_ac(name, dev), d, 5, 1, monkeypatch, dev, accumulate=False)[0]
    whole, _, rows = _grad_errors(free["grads"], acc["grads"])
    print(f"{name}: autograd.grad vs adopted .grad: whole {whole:.2e}, worst tensor {rows[0][1]} {rows[0][0]:.1e}")
    assert free["loss"] == acc["loss"]
    assert whole < AUTOGRAD_WHOLE_TOL and rows[0][0] < AUTOGRAD_TENSOR_TOL, (whole, rows[0])


# ------------------------------------------------------------------------------------------------ default widths unchanged
@gpu
def test_default_policy_launch_counts_unchanged(dev):
    cfg = O.ActorCriticCfg()
    ac = _native_ac(cfg, O.seeded_actor_critic_state_dict(cfg, 616), dev)
    obs, hx, cx, g_out = _node_args(cfg, dev, 32, 4)
    lib = _lib.lib()
    _Node(ac, obs, hx, cx)   # set_weights and first-call work outside the counted window
    torch.cuda.synchronize()
    lib.dmd_launch_count(1)
    n = _Node(ac, obs, hx, cx)
    fwd = lib.dmd_launch_count(1)
    n.backward(g_out, torch.empty(ac._grad_views_layout()[2], device=dev))
    bwd = lib.dmd_launch_count(1)
    print(f"default policy at B=32: {fwd} launches per forward, {bwd} per backward")
    assert (fwd, bwd) == (DEFAULT_FWD_LAUNCHES, DEFAULT_BWD_LAUNCHES)
