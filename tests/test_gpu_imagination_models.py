"""The two executors of the imagination update (bench.py cfg 3) at the shapes and call patterns it runs them with, against the
reference-pinned oracle in float64.

Actor-critic: `ActorCritic.forward()` + `backward()` through the env loop with DEAD-ENV BURN-IN (env_loop.py:53-56: the dead
envs' recurrent state is burnt in WITH gradient on the new episode's context frames and index-put back into the batch).  Those
burn-in calls are native autograd nodes at B = number of dead envs (down to 1) whose backward receives only g_hx / g_cx.
Checked on the reference's own burn-in run (tests/golden/actor_critic_burnin.npz), at the benchmark shape (32 envs x 15
steps, two updates with the truncated-BPTT carry between them), on the non-accumulating path `torch.autograd.grad` needs, and
kernel by kernel for the head-gradient combinations burn-in produces.

Reward/termination model: the call sequence WorldModelEnv makes (a 96-row burn-in on every pool refill, 32-row single steps
carrying (hx, cx), fresh burn-in states spliced into the rows of dead envs), an odd batch with several time steps, weights
updated in place and moved to new addresses, and a second configuration (64 channels with a projection, attention in a level).

The CPU tests at the end show that each plausible mistake of these call patterns misses the bounds used here by at least 10x."""
import os

import numpy as np
import pytest
import torch
from torch.distributions.categorical import Categorical

from oracle import torch_oracle as O
from oracle.make_golden import BURNIN_T, frames_from_u8, load_actor_critic_burnin

gpu = pytest.mark.gpu

LOGITS_TOL = 1e-3     # actor logits and recurrent state per step
VAL_TOL = 2e-3        # the scalar value head: one 512-term dot product with cancellation (tests/test_actor_critic.py)
GRAD_TOL = 1e-3       # whole gradient, relative L2 over all parameters
TENSOR_TOL = 4e-3     # one gradient tensor (or negligible against the whole gradient) ...
PER_TENSOR_CAP = 5e-3  # ... and never more than this (tests/test_gpu_training.py)
REW_LOGITS_TOL = 2e-3  # reward / termination logits (tests/test_gpu_rew_end.py)
REW_STATE_TOL = 1e-3   # its LSTM state


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


# ================================================================================================ actor-critic
class _BurninEnv:
    """Scripted environment: pre-generated observations, rewards and flags (the action is ignored); with every death it
    returns `final_observation` and, like WorldModelEnv.step, `burnin_obs` (k, 3, C, H, W) for the k dead envs."""

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


def _native_ac(sd, dev):
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig

    cfg = O.ActorCriticCfg()
    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    ac.load_state_dict(sd)
    return ac.to(dev).train()


def _run_native_updates(ac, d, T, n_updates, monkeypatch, dev, accumulate=True):
    """n_updates calls of ActorCritic.forward() on the scripted env (actions replayed from d["act"] through
    Categorical.sample), each followed by backward: loss.backward() into .grad, or torch.autograd.grad without accumulation.
    Returns per update: loss, logs, the rollout's logits / values, and the gradients by parameter name."""
    from diamond_b200.models.actor_critic import ActorCriticLossConfig

    lc = O.ActorCriticLossCfg(backup_every=T)
    ac.setup_training(_BurninEnv(d, dev), ActorCriticLossConfig(lc.backup_every, lc.gamma, lc.lambda_, lc.weight_value_loss,
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
            assert all(p.grad is None for p in ac.parameters()), "torch.autograd.grad must not write .grad"
            grads = {k: g.detach().cpu() for k, g in zip(names, gs)}
        torch.cuda.synchronize()
        rollout = captured[-1]
        out.append(dict(loss=float(loss.detach()), logs={k: float(v) for k, v in logs.items()}, logits=rollout[5].detach().cpu(),
                        val=rollout[6].detach().cpu(), grads=grads))
    monkeypatch.undo()
    assert step[0] == n_updates * T
    return out


def _shift(dct, t0, T, dtype):
    return {t - t0: v.to(dtype) for t, v in dct.items() if t0 <= t < t0 + T}


def _oracle_update(d, sd, t0, T, state=None, dtype=torch.float64, burnin=True):
    """The oracle rollout of steps [t0, t0 + T) (continuing from `state`, detached) + the reference loss and its gradient."""
    cfg = O.ActorCriticCfg()
    sl = slice(t0, t0 + T)
    hx, cx = state if state is not None else (None, None)
    logits, val, vb, (hx, cx) = O.actor_critic_rollout(
        d["obs_seq"][t0:t0 + T + 1].to(dtype), d["end"][sl], d["trunc"][sl], _shift(d["final_obs"], t0, T, dtype), sd, cfg, hx, cx,
        burnin_obs=_shift(d["burnin_obs"], t0, T, dtype) if burnin else None, return_state=True)
    loss, metrics = O.actor_critic_loss(logits, val, d["act"][:, sl], d["rew"][sl].t().to(dtype), d["end"][sl].t().to(dtype),
                                        d["trunc"][sl].t().to(dtype), vb, O.ActorCriticLossCfg(backup_every=T))
    gs = torch.autograd.grad(loss, list(sd.values()))
    return dict(loss=float(loss.detach()), logs={k: float(v) for k, v in metrics.items()}, logits=logits.detach(), val=val.detach(),
                grads=dict(zip(sd, gs)), state=(hx.detach(), cx.detach()))


def _oracle_params(seed, dtype=torch.float64):
    return {k: v.to(dtype).requires_grad_(True) for k, v in O.seeded_actor_critic_state_dict(O.ActorCriticCfg(), seed).items()}


def _grad_errors(grads, ref):
    """(whole-gradient relative L2 error, |G|, rows (relative error, name, |g|) sorted worst first)."""
    num = den = 0.0
    rows = []
    for k, r in ref.items():
        r = r.double()
        dlt = grads[k].double() - r
        num += float(dlt.pow(2).sum()); den += float(r.pow(2).sum())
        rows.append((float(dlt.norm() / r.norm().clamp_min(1e-30)), k, float(r.norm())))
    return (num / den) ** 0.5, den ** 0.5, sorted(rows, reverse=True)


def _check_update(label, nat, ref):
    """Per-step logits / values, loss, metrics, whole gradient and every tensor; prints the errors and the worst tensors."""
    T = ref["logits"].size(1)
    e_log = [_rel(nat["logits"][:, t], ref["logits"][:, t]) for t in range(T)]
    e_val = [_rel(nat["val"][:, t], ref["val"][:, t]) for t in range(T)]
    whole, total, rows = _grad_errors(nat["grads"], ref["grads"])
    e_loss = abs(nat["loss"] - ref["loss"]) / abs(ref["loss"])
    print(f"{label}: logits per step " + " ".join(f"{e:.1e}" for e in e_log))
    print(f"{label}: values per step " + " ".join(f"{e:.1e}" for e in e_val))
    print(f"{label}: worst logits {max(e_log):.2e}, values {max(e_val):.2e}, loss native {nat['loss']:.6f} oracle "
          f"{ref['loss']:.6f} (rel {e_loss:.2e}), whole gradient {whole:.2e}")
    print(f"{label}: worst tensors " + ", ".join(f"{k} {e:.2e} (|g| {n:.2e})" for e, k, n in rows[:5]))
    assert max(e_log) < LOGITS_TOL, e_log
    assert max(e_val) < VAL_TOL, e_val
    assert abs(nat["loss"] - ref["loss"]) <= 2e-3 * abs(ref["loss"]) + 1e-5, (nat["loss"], ref["loss"])
    for k, v in ref["logs"].items():
        assert abs(nat["logs"][k] - v) <= 3e-3 * abs(v) + 1e-5, (k, nat["logs"][k], v)
    assert whole < GRAD_TOL, whole
    for e, k, n in rows:
        assert e < TENSOR_TOL or e * n < 1e-4 * total, (k, e, n, total)
        assert e < PER_TENSOR_CAP, (k, e, n, total)


@gpu
def test_actor_critic_burnin_matches_reference(golden_dir, monkeypatch):
    """The reference's own forward + backward with burn-in (6 envs x 6 steps: a death at t = 0, lone and paired deaths, one
    env dying three times, all envs truncated at once, a death on the last step): loss, metrics and gradient norms against
    the golden, and every gradient tensor against the float64 oracle."""
    dev = _dev()
    g = np.load(os.path.join(golden_dir, "actor_critic_burnin.npz"))
    d = load_actor_critic_burnin(g)
    nat = _run_native_updates(_native_ac(O.seeded_actor_critic_state_dict(O.ActorCriticCfg(), 557), dev), d, BURNIN_T, 1, monkeypatch, dev)[0]
    print(f"burn-in golden: loss native {nat['loss']:.6f} reference {float(g['loss']):.6f}")
    assert abs(nat["loss"] - float(g["loss"])) <= 2e-3 * abs(float(g["loss"])) + 1e-5
    for k, v in zip(g["metric_keys"], g["metric_vals"]):
        assert abs(nat["logs"][str(k)] - float(v)) <= 3e-3 * abs(float(v)) + 1e-5, (k, nat["logs"][str(k)], float(v))
    keys = [str(k) for k in g["grad_keys"]]
    norms = np.array([float(nat["grads"][k].double().norm()) for k in keys])
    ref_n = g["grad_norms"]
    tot = float(np.sqrt((ref_n ** 2).sum()))
    assert np.all(np.abs(norms - ref_n) <= 4e-3 * ref_n + 1e-4 * tot), float(np.max(np.abs(norms - ref_n) / ref_n))
    torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))
    _check_update("burn-in golden", nat, _oracle_update(d, _oracle_params(557), 0, BURNIN_T))


# The benchmark shape: 32 envs, backup_every = 15, two updates (steps 0-14 and 15-29).  Deaths per step; every death returns
# 3 burn-in frames, i.e. 3 more autograd nodes at B = number of dead envs.  Live nodes per update: 15 + 3 x 8 = 39 and
# 15 + 3 x 6 = 33, under the actor-critic's workspace-pool cap of 64.
AC_B, AC_T, AC_SEED = 32, 15, 558
AC_DEATHS = {0: [5], 2: [1, 9, 30], 4: [17], 5: [3, 22], 7: [0, 8, 12, 19, 27, 31], 9: [5], 11: [2, 14, 25, 29], 14: list(range(AC_B)),
             16: [7], 18: [11, 20], 21: [5, 6, 13, 26, 28], 23: [31], 26: [4, 10, 16], 29: [18]}


def _bench_rollout_data():
    """Frames on the 1/255 grid, rewards, the AC_DEATHS flags (every env truncated at t = 14, the others alternate between
    termination and truncation), final / burn-in frames of the dead envs and pre-drawn actions, from a seed."""
    rng = np.random.default_rng(2025)
    steps, img = 2 * AC_T, (3, 64, 64)
    end = torch.zeros(steps, AC_B, dtype=torch.long)
    trunc = torch.zeros(steps, AC_B, dtype=torch.long)
    final_obs, burnin_obs = {}, {}
    for t, envs in AC_DEATHS.items():
        for e in envs:
            (trunc if t == AC_T - 1 or (t + e) % 3 == 0 else end)[t, e] = 1
        final_obs[t] = frames_from_u8(rng.integers(0, 256, size=(len(envs),) + img, dtype=np.uint8))
        burnin_obs[t] = frames_from_u8(rng.integers(0, 256, size=(len(envs), 3) + img, dtype=np.uint8))
    return dict(obs_seq=frames_from_u8(rng.integers(0, 256, size=(steps + 1, AC_B) + img, dtype=np.uint8)),
                rew=torch.from_numpy(rng.choice([-1.0, 0.0, 0.0, 2.0], size=(steps, AC_B)).astype(np.float32)), end=end, trunc=trunc,
                final_obs=final_obs, burnin_obs=burnin_obs, act=torch.from_numpy(rng.integers(0, 4, size=(AC_B, steps))))


@gpu
def test_actor_critic_benchmark_shape_two_updates_match_oracle(monkeypatch):
    """32 envs x 15 steps with burn-in (nodes of 1 to 32 rows), then a second update continuing from the carried, detached
    (hx, cx): per-step logits and values, loss, metrics, the whole gradient and each tensor against the float64 oracle, which
    carries its own state into its second update."""
    dev = _dev()
    d = _bench_rollout_data()
    assert AC_T + 3 * sum(1 for t in AC_DEATHS if t < AC_T) < 64 and AC_T + 3 * sum(1 for t in AC_DEATHS if t >= AC_T) < 64
    nat = _run_native_updates(_native_ac(O.seeded_actor_critic_state_dict(O.ActorCriticCfg(), AC_SEED), dev), d, AC_T, 2, monkeypatch, dev)
    torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))
    sd = _oracle_params(AC_SEED)
    ref1 = _oracle_update(d, sd, 0, AC_T)
    _check_update("B=32 update 1", nat[0], ref1)
    ref2 = _oracle_update(d, sd, AC_T, AC_T, state=ref1["state"])
    _check_update("B=32 update 2 (carried state)", nat[1], ref2)


@gpu
def test_actor_critic_autograd_grad_matches_accumulated_grad(golden_dir, monkeypatch):
    """accumulate_native_grads = False (every node returns its parameter gradients to autograd, which torch.autograd.grad
    needs) on the burn-in rollout against the natively accumulated .grad of the same rollout.  The two differ only in the
    order of fp32 additions across nodes and in the fp64 atomics of the GroupNorm sums: bound 1e-6 on the whole gradient,
    1e-5 on each tensor (measured on an H100 SXM, 700 W: 1.4e-7 and 1.9e-6, encoder.encoder.0.weight)."""
    dev = _dev()
    d = load_actor_critic_burnin(np.load(os.path.join(golden_dir, "actor_critic_burnin.npz")))
    sd = O.seeded_actor_critic_state_dict(O.ActorCriticCfg(), 557)
    acc = _run_native_updates(_native_ac(sd, dev), d, BURNIN_T, 1, monkeypatch, dev, accumulate=True)[0]
    free = _run_native_updates(_native_ac(sd, dev), d, BURNIN_T, 1, monkeypatch, dev, accumulate=False)[0]
    whole, _, rows = _grad_errors(free["grads"], acc["grads"])
    print(f"autograd.grad vs accumulated .grad: whole {whole:.2e}, worst tensors", [(k, f"{e:.1e}") for e, k, _ in rows[:3]])
    assert free["loss"] == acc["loss"]
    assert whole < 1e-6, whole
    assert rows[0][0] < 1e-5, rows[0]


# ------------------------------------------------------------------------------------------------ heads + LSTM cell backward
def _ref_heads_cell(gates, c_in, wa, ba, wc, bc, g_hx, g_cx, g_logits, g_val):
    """float64 autograd of LSTMCell (torch gate order) + actor / critic heads: gradients wrt the gate pre-activations, the
    incoming cell state, the actor bias and the critic weight / bias.  Absent output gradients are absent terms."""
    x, c0, ba_, wc_, bc_ = [t.double().detach().requires_grad_() for t in (gates, c_in, ba, wc, bc)]
    i, f, gg, o = x.chunk(4, dim=1)
    c1 = torch.sigmoid(f) * c0 + torch.sigmoid(i) * torch.tanh(gg)
    h1 = torch.sigmoid(o) * torch.tanh(c1)
    total = h1.sum() * 0
    if g_hx is not None:
        total = total + (h1 * g_hx.double()).sum()
    if g_cx is not None:
        total = total + (c1 * g_cx.double()).sum()
    if g_logits is not None:
        total = total + ((h1 @ wa.double().t() + ba_) * g_logits.double()).sum()
    if g_val is not None:
        total = total + ((h1 @ wc_.view(-1, 1) + bc_).squeeze(1) * g_val.double()).sum()
    grads = torch.autograd.grad(total, (x, c0, ba_, wc_, bc_), allow_unused=True, materialize_grads=True)
    return h1.detach(), grads


@gpu
@pytest.mark.parametrize("b", [1, 5])
@pytest.mark.parametrize("case", ["state_only", "heads_no_g_hx", "actor_no_g_hx", "critic_no_g_hx"])
def test_heads_and_cell_bwd_burnin_combinations(b, case):
    """What a burn-in node's backward receives: g_hx and g_cx without any head gradient ("state_only", its logits and value
    are discarded); and head gradients without g_hx (a step whose new state feeds nothing that needs a gradient), with one or
    both heads.  heads_bwd then lstm_cell_bwd against float64 autograd; absent heads leave their parameter gradients alone."""
    dev = _dev()
    from diamond_b200 import ops

    g = torch.Generator().manual_seed(b * 7 + len(case))
    hd, a = 512, 4
    gates, c_in = 2 * torch.randn(b, 4 * hd, generator=g), torch.randn(b, hd, generator=g)
    wa, ba = torch.randn(a, hd, generator=g) / 20, torch.randn(a, generator=g)
    wc, bc = torch.randn(1, hd, generator=g) / 20, torch.randn(1, generator=g)
    g_hx = torch.randn(b, hd, generator=g) if case == "state_only" else None
    g_cx = torch.randn(b, hd, generator=g) if case == "state_only" else None
    g_logits = torch.randn(b, a, generator=g) if case in ("heads_no_g_hx", "actor_no_g_hx") else None
    g_val = torch.randn(b, generator=g) if case in ("heads_no_g_hx", "critic_no_g_hx") else None
    h1, (r_dg, r_gc, r_dba, r_dwc, r_dbc) = _ref_heads_cell(gates, c_in, wa, ba, wc, bc, g_hx, g_cx, g_logits, g_val)
    pre = [torch.randn(a, generator=g), torch.randn(1, hd, generator=g), torch.randn(1, generator=g)]
    dba, dwc, dbc = [p.to(dev).clone() for p in pre]
    to = lambda t: None if t is None else t.to(dev)  # noqa: E731
    g_h = ops.heads_bwd(to(g_hx), to(g_logits), to(g_val), h1.float().to(dev), wa.to(dev), wc.to(dev), dba, dwc, dbc)
    dg, gc = ops.lstm_cell_bwd(gates.to(dev), c_in.to(dev), g_h, to(g_cx))
    errs = {"dgates": _rel(dg, r_dg), "g_c_in": _rel(gc, r_gc)}
    if g_logits is not None:
        errs["dba"] = _rel(dba.cpu().double() - pre[0].double(), r_dba)
    else:
        assert torch.equal(dba.cpu(), pre[0])
    if g_val is not None:
        errs["dWc"] = _rel(dwc.cpu().double() - pre[1].double(), r_dwc)
        errs["dbc"] = _rel(dbc.cpu().double() - pre[2].double(), r_dbc)
    else:
        assert torch.equal(dwc.cpu(), pre[1]) and torch.equal(dbc.cpu(), pre[2])
    print(f"heads + cell bwd B={b} {case}:", {k: f"{v:.1e}" for k, v in errs.items()})
    assert max(errs.values()) < 1e-5, errs


# ================================================================================================ reward / termination model
REW_CFGS = {
    "default": O.RewEndCfg(),
    # a 32 -> 64 channel step (level 2's first ResBlock has a 1x1 projection), attention inside the last level (8 x 8 = 64
    # tokens at 64 channels), conditioning width 64
    "wide_attn": O.RewEndCfg(cond_channels=64, channels=[32, 32, 64, 64], attn_depths=[0, 0, 0, 1]),
}
REW_B, REW_STEPS, REW_SEED = 32, 15, 779
# before single step k: the envs that died at step k - 1 take fresh burn-in states from the pool (WorldModelEnv.reset_dead)
REW_SPLICES = {5: [3, 17, 30], 9: [0, 8, 21, 22], 12: [5]}


def _rew_end_model(cfg, sd, dev):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig

    m = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                      list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
    m.load_state_dict(sd)
    return m.to(dev).eval()


def _rew_end_data(seed):
    """Two pool batches (32 x 4 frames, 3 actions) for the refill burn-ins and 32 envs x 16 frames / 15 actions to step on."""
    rng = np.random.default_rng(seed)
    img = (3, 64, 64)
    return dict(pool=[(frames_from_u8(rng.integers(0, 256, size=(REW_B, 4) + img, dtype=np.uint8)),
                       torch.from_numpy(rng.integers(0, 4, size=(REW_B, 3)))) for _ in range(2)],
                frames=frames_from_u8(rng.integers(0, 256, size=(REW_B, REW_STEPS + 1) + img, dtype=np.uint8)),
                act=torch.from_numpy(rng.integers(0, 4, size=(REW_B, REW_STEPS))))


def _rew_end_sequence(predict, d, splices=REW_SPLICES, skip_state_at=None, steps=REW_STEPS):
    """The calls WorldModelEnv makes, through predict(obs, act, next_obs, hx_cx) -> (rew, end, (hx, cx)): a refill burn-in
    (t = 3, no state) whose states start every env; `steps` single steps carrying (hx, cx); before the steps in `splices` the
    listed rows take the next fresh states of the pool, the first such request refilling it (a second 96-row burn-in).
    Returns [(label, logits [b, t, 5], hx, cx)] per call.  skip_state_at: a step called without its state (a mistake)."""
    calls = []

    def burn(i):
        obs, act = d["pool"][i]
        lr, le, hc = predict(obs[:, :3], act, obs[:, 1:4], None)
        calls.append((f"refill {i} (96 rows)", torch.cat([lr, le], -1), hc[0], hc[1]))
        return hc

    hx, cx = burn(0)
    pool, cursor = None, 0
    for k in range(steps):
        if k in splices:
            rows = splices[k]
            if pool is None:
                pool = burn(1)
            hx, cx = hx.clone(), cx.clone()
            hx[:, rows] = pool[0][:, cursor:cursor + len(rows)]
            cx[:, rows] = pool[1][:, cursor:cursor + len(rows)]
            cursor += len(rows)
        f, a = d["frames"], d["act"]
        lr, le, (hx, cx) = predict(f[:, k:k + 1], a[:, k:k + 1], f[:, k + 1:k + 2], None if k == skip_state_at else (hx, cx))
        calls.append((f"step {k}" + (" (splice)" if k in splices else ""), torch.cat([lr, le], -1), hx, cx))
    return calls


def _native_predict(m, dev):
    def predict(obs, act, nxt, hc):
        return m.predict_rew_end(obs.to(dev), act.to(dev), nxt.to(dev), hc)
    return predict


def _oracle_predict(sd, cfg, dtype=torch.float64):
    sd = {k: v.to(dtype) for k, v in sd.items()}

    def predict(obs, act, nxt, hc):
        return O.predict_rew_end(obs.to(dtype), act, nxt.to(dtype), sd, cfg, hc)
    return predict


def _call_errors(got, ref):
    return [(lab, _rel(gl, rl), max(_rel(gh, rh), _rel(gc, rc))) for (lab, gl, gh, gc), (_, rl, rh, rc) in zip(got, ref)]


@gpu
@pytest.mark.parametrize("name", list(REW_CFGS))
def test_rew_end_env_call_sequence_matches_oracle(name):
    """Rows alternate 96 -> 32 -> 96 -> 32 on one workspace (the encoder plan is rebuilt each time), the state is carried
    over 15 steps and fresh burn-in states are spliced into some rows: every call's logits (2e-3) and state (1e-3) against
    the float64 oracle, which carries its own state.  The error is printed per call so that drift shows.

    The state error sits close to its bound by design, not by drift: measured on an H100 SXM (700 W) it is 9.0e-4 to 9.7e-4 on
    every call of the default config (7.1e-4 for the wide one), and the oracle with its 3x3 conv operands rounded to fp16, as
    the kernels round them, is off by 1.07e-3 (hx) / 9.6e-4 (cx) on the first burn-in."""
    dev = _dev()
    cfg = REW_CFGS[name]
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), REW_SEED)
    d = _rew_end_data(REW_SEED + 1)
    m = _rew_end_model(cfg, sd, dev)
    got = _rew_end_sequence(_native_predict(m, dev), d)
    torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))
    errs = _call_errors(got, _rew_end_sequence(_oracle_predict(sd, cfg), d))
    for lab, el, es in errs:
        print(f"rew_end {name} {lab:20s} logits {el:.2e}  state {es:.2e}")
    print(f"rew_end {name}: worst logits {max(e[1] for e in errs):.2e}, worst state {max(e[2] for e in errs):.2e}")
    assert len(errs) == 2 + REW_STEPS
    for lab, el, es in errs:
        assert el < REW_LOGITS_TOL and es < REW_STATE_TOL, (lab, el, es)


def _odd_inputs(b, t, seed, with_state):
    rng = np.random.default_rng(seed)
    frames = frames_from_u8(rng.integers(0, 256, size=(b, t + 1, 3, 64, 64), dtype=np.uint8))
    act = torch.from_numpy(rng.integers(0, 4, size=(b, t)))
    hc = None
    if with_state:
        hc = tuple(torch.from_numpy(0.3 * rng.standard_normal((1, b, 512))).float() for _ in range(2))
    return frames[:, :t], act, frames[:, 1:], hc


@gpu
@pytest.mark.parametrize("b,t,with_state", [(1, 1, False), (1, 1, True), (5, 4, True)])
def test_rew_end_small_and_odd_batches_match_oracle(b, t, with_state):
    """One row; and 5 envs x 4 steps, where rows are packed time-major (row = k * b + n) and the LSTM walks b-row blocks."""
    dev = _dev()
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), REW_SEED)
    obs, act, nxt, hc = _odd_inputs(b, t, 31 + b * t, with_state)
    m = _rew_end_model(cfg, sd, dev)
    lr, le, (hx, cx) = m.predict_rew_end(obs.to(dev), act.to(dev), nxt.to(dev), None if hc is None else tuple(s.to(dev) for s in hc))
    rr, re, (rhx, rcx) = _oracle_predict(sd, cfg)(obs, act, nxt, None if hc is None else tuple(s.double() for s in hc))
    el = _rel(torch.cat([lr, le], -1), torch.cat([rr, re], -1))
    es = max(_rel(hx, rhx), _rel(cx, rcx))
    per_step = [_rel(torch.cat([lr, le], -1)[:, k], torch.cat([rr, re], -1)[:, k]) for k in range(t)]
    print(f"rew_end b={b} t={t} state={with_state}: logits {el:.2e} (per step {['%.1e' % e for e in per_step]}), state {es:.2e}")
    assert lr.shape == (b, t, 3) and le.shape == (b, t, 2) and hx.shape == (1, b, 512)
    assert el < REW_LOGITS_TOL and es < REW_STATE_TOL, (el, per_step, es)


@gpu
def test_rew_end_follows_weights_updated_in_place_and_moved():
    """p.mul_(1.01) in place: the next call follows the oracle on the new weights and differs from the old outputs.  Moved
    to the CPU and back (the old device copies kept alive and overwritten with NaN, so every parameter address changes and a
    stale pointer would show): the same results as a fresh model on those weights."""
    dev = _dev()
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), REW_SEED)
    obs, act, nxt, hc = _odd_inputs(5, 4, 77, True)
    m = _rew_end_model(cfg, sd, dev)

    def run(model):
        lr, le, (hx, cx) = model.predict_rew_end(obs.to(dev), act.to(dev), nxt.to(dev), tuple(s.to(dev) for s in hc))
        return torch.cat([lr, le], -1).cpu(), hx.cpu(), cx.cpu()

    old = run(m)
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(1.01)
    new = run(m)
    sd2 = {k: v * 1.01 for k, v in sd.items()}     # the same fp32 products the module now holds
    ref = _oracle_predict(sd2, cfg)(obs, act, nxt, tuple(s.double() for s in hc))
    e_new = (_rel(new[0], torch.cat(ref[:2], -1)), max(_rel(new[1], ref[2][0]), _rel(new[2], ref[2][1])))
    moved_by = _rel(new[0], old[0])
    print(f"rew_end after p.mul_(1.01): logits {e_new[0]:.2e}, state {e_new[1]:.2e}; logits moved by {moved_by:.2e}")
    assert e_new[0] < REW_LOGITS_TOL and e_new[1] < REW_STATE_TOL, e_new
    assert moved_by > 10 * REW_LOGITS_TOL, moved_by

    keep = [t for t in m.state_dict().values()]     # the current device copies stay allocated ...
    before = {k: t.data_ptr() for k, t in m.state_dict().items()}
    m.cpu()
    m.cuda(dev)
    for t in keep:                                  # ... and are poisoned once the module no longer owns them
        t.fill_(float("nan"))
    assert all(t.data_ptr() != before[k] for k, t in m.state_dict().items())
    moved = run(m)
    fresh = run(_rew_end_model(cfg, {k: v.cpu() for k, v in m.state_dict().items()}, dev))
    errs = [_rel(a, b) for a, b in zip(moved, fresh)]
    print(f"rew_end moved vs fresh model: {['%.1e' % e for e in errs]}")
    assert all(torch.isfinite(t).all() for t in moved)
    assert max(errs) < 1e-5, errs


# ================================================================================================ CPU: the bounds have teeth
def _worst_ratio(label, bad, ref):
    """How far a mistaken actor-critic update misses the bounds above (per-step logits, values, whole gradient)."""
    T = ref["logits"].size(1)
    e = {"logits": max(_rel(bad["logits"][:, t], ref["logits"][:, t]) for t in range(T)) / LOGITS_TOL,
         "values": max(_rel(bad["val"][:, t], ref["val"][:, t]) for t in range(T)) / VAL_TOL,
         "gradient": _grad_errors(bad["grads"], ref["grads"])[0] / GRAD_TOL}
    print(f"mistake '{label}': error / bound " + ", ".join(f"{k} {v:.1f}x" for k, v in e.items()))
    return max(e.values())


def test_imagination_mistakes_exceed_tolerance(monkeypatch):
    """Each mistake below, made by the oracle at the shapes of the GPU tests above, misses their bounds by at least 10x
    (fp32 oracle: its own round-off is far below the bounds)."""
    torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))
    f32 = torch.float32
    # ---- actor-critic, first update of the benchmark shape
    d = _bench_rollout_data()
    ref = _oracle_update(d, _oracle_params(AC_SEED, f32), 0, AC_T, dtype=f32)
    assert _worst_ratio("burn-in skipped", _oracle_update(d, _oracle_params(AC_SEED, f32), 0, AC_T, dtype=f32, burnin=False), ref) > 10
    # burn-in results written to the wrong dead envs (rolled by one among them on every step with several deaths)
    rolled = dict(d, burnin_obs={t: v.roll(1, 0) for t, v in d["burnin_obs"].items()})
    assert _worst_ratio("burn-in on the wrong rows", _oracle_update(rolled, _oracle_params(AC_SEED, f32), 0, AC_T, dtype=f32), ref) > 10
    # burn-in run without gradient: the forward is unchanged, the gradient through the burnt-in state is lost
    burn_ptrs = {v.untyped_storage().data_ptr() for v in d["burnin_obs"].values()}
    real = O.predict_act_value

    def no_grad_burnin(obs, hx, cx, sd, cfg):
        if obs.untyped_storage().data_ptr() in burn_ptrs:
            with torch.no_grad():
                return real(obs, hx, cx, sd, cfg)
        return real(obs, hx, cx, sd, cfg)

    monkeypatch.setattr(O, "predict_act_value", no_grad_burnin)
    bad = _oracle_update(d, _oracle_params(AC_SEED, f32), 0, AC_T, dtype=f32)   # float32 frames: _shift keeps their storage
    monkeypatch.undo()
    assert torch.equal(bad["logits"], ref["logits"])
    assert _worst_ratio("burn-in without gradient", bad, ref) > 10

    # ---- reward / termination model
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), REW_SEED)
    pred = _oracle_predict(sd, cfg, f32)
    # rows packed batch-major where the LSTM reads them time-major (b = 5, t = 4)
    obs, act, nxt, hc = _odd_inputs(5, 4, 31 + 20, True)
    good = torch.cat(pred(obs, act, nxt, hc)[:2], -1)

    def bm(x):   # the (b, t) grid read in the other order
        return x.transpose(0, 1).reshape(x.shape)
    wrong = torch.cat(pred(bm(obs), bm(act), bm(nxt), hc)[:2], -1)
    e_order = _rel(wrong, good) / REW_LOGITS_TOL
    print(f"mistake 'rew-end rows batch-major': logits error / bound {e_order:.1f}x")
    assert e_order > 10
    # the state not carried into one step; a splice written to the wrong envs (b = 32).  Only the calls up to the affected
    # one run, the splice of step 5 being the first.
    d = _rew_end_data(REW_SEED + 1)
    good = _rew_end_sequence(pred, d, steps=6)
    for label, kw in (("state not carried into step 3", dict(skip_state_at=3)),
                      ("splice written to the wrong envs", dict(splices={5: [4, 18, 31]}))):
        errs = _call_errors(_rew_end_sequence(pred, d, steps=6, **kw), good)
        ratio = max(max(el / REW_LOGITS_TOL, es / REW_STATE_TOL) for _, el, es in errs)
        print(f"mistake '{label}': worst call error / bound {ratio:.1f}x")
        assert ratio > 10
