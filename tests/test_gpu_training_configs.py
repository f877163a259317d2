"""Training across the model configurations the native entry points accept (oracle/training_configs.py): the backward plan's
topology-dependent decisions (first writer assigns, later writers accumulate; which concat source carries the identity
residual; per-source dgrad packs; projections 32 -> 64 and 64 -> 32; a one-level U-Net; a three-pass conv_in; more than 8
output channels) and the actor-critic's immediate-mode backward at levels without a max-pool.

Every case trains through the public Python surface with its random draws and actions replayed, and is checked against the
oracle's float64 autograd.  The bounds come from the kernels' operand rounding emulated at the case's own inputs
(oracle/fp16_emulation.py grad_errors, float64):
  - loss within 2e-3 relative;
  - whole gradient (relative L2 over every parameter) within WHOLE_MARGIN x the emulation's, a bound that may not exceed
    WHOLE_CAP;
  - every tensor within TENSOR_MARGIN x its emulated error, or negligible against the whole gradient
    (e |g| < 1e-4 |G|), and never above PER_TENSOR_CAP;
  - a second identical step within RUN_TO_RUN_SHARE x the emulated whole-gradient error (atomic-addition order);
  - every .grad finite.
The CPU tests below check that the cases reach what they are meant to reach, that plausible plan mistakes miss these bounds
by at least 10x, and that the float64 oracle equals the unmodified reference at D1 and D4."""
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import fp16_emulation as E
from oracle import rew_end_training as RT
from oracle import torch_oracle as O
from oracle import training_configs as TC

gpu = pytest.mark.gpu

WHOLE_MARGIN = 1.25      # the "budget + 25 %" of tests/test_gpu_training.py
WHOLE_CAP = 2e-3
TENSOR_MARGIN = 2.0
PER_TENSOR_CAP = 5e-3    # as tests/test_gpu_training.py
# A second identical step differs by the order of fp32 / fp64 atomic additions.  Where three or more blocks add into one sum
# (the per-(image, channel) sums of the norm backward at these small batches), the fp32 result moves by an ulp, and the fp16
# rounding of the next conv's gradient operand turns that into an occasional fp16 ulp: measured on an H100 80GB HBM3 (700 W),
# 2e-5 .. 7e-5 of the whole gradient, at most 0.14 of the emulated rounding error.  The bound is a quarter of it.
RUN_TO_RUN_SHARE = 0.25
CONTROL_MARGIN = 10.0    # a negative control must miss its case's whole-gradient bound by this factor
F64 = torch.float64


def _loss_scale_exp():
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "diamond_b200.h")) as f:
        return int(re.search(r"#define DMD_LOSS_SCALE_EXP (\d+)", f.read()).group(1))


def _threads():
    torch.set_num_threads(min(16, max(1, os.cpu_count() or 1)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _leaves(sd, frozen=("noise_emb.weight",)):
    for k, v in sd.items():
        if k not in frozen:
            v.requires_grad_(True)
    return sd


# ------------------------------------------------------------------------------------------------ float64 losses
def _denoiser_loss_fn(c):
    obs, act, mask, draws = TC.denoiser_inputs(c)
    obs64, draws64 = obs.to(F64), [tuple(t.to(F64) for t in d) for d in draws]
    cfg = O.DenoiserCfg(inner=c["inner"])
    return lambda sd: O.denoiser_loss(obs64, act, mask, draws64, sd, cfg, O.SigmaDistCfg())


def _denoiser_sd(c):
    return _leaves(O.seeded_state_dict(O.inner_model_shapes(c["inner"]), c["wseed"], dtype=F64))


def _rew_end_loss_fn(c):
    obs, act, rew, end, mask, final_obs = TC.rew_end_inputs(c)
    fo64 = {i: f.to(F64) for i, f in final_obs.items()}
    return lambda sd: RT.rew_end_loss(obs.to(F64), act, rew.to(F64), end, mask, fo64, sd, c["cfg"])[0]


def _rew_end_sd(c):
    return _leaves(O.seeded_state_dict(O.rew_end_shapes(c["cfg"]), c["wseed"], dtype=F64), ())


def _actor_critic_loss_fn(c):
    obs_seq, rew, end, trunc, final_obs, act = TC.actor_critic_inputs(c)
    fo64 = {t: f.to(F64) for t, f in final_obs.items()}
    lc = O.ActorCriticLossCfg(backup_every=c["T"])

    def loss(sd):
        logits, val, vb = O.actor_critic_rollout(obs_seq.to(F64), end, trunc, fo64, sd, c["cfg"])
        return O.actor_critic_loss(logits, val, act, rew.t().to(F64), end.t().to(F64), trunc.t().to(F64), vb, lc)[0]
    return loss


def _actor_critic_sd(c):
    return {k: v.to(F64).requires_grad_(True) for k, v in O.seeded_actor_critic_state_dict(c["cfg"], c["wseed"]).items()}


def _case(name):
    """(loss closure, float64 state dict, stream predicate, output conv, loss-scale exponent) of a case."""
    if name in TC.DENOISER_CASES:
        c = TC.DENOISER_CASES[name]
        sd = _denoiser_sd(c)
        return _denoiser_loss_fn(c), sd, E.denoiser_stream(sd), "conv_out.weight", _loss_scale_exp()
    if name in TC.REW_END_CASES:
        c = TC.REW_END_CASES[name]
        sd = _rew_end_sd(c)
        return _rew_end_loss_fn(c), sd, E.rew_end_stream(sd), None, None
    c = TC.ACTOR_CRITIC_CASES[name]
    sd = _actor_critic_sd(c)
    return _actor_critic_loss_fn(c), sd, E.actor_critic_stream(sd), None, None


def _budget(name):
    """The emulation at the case's inputs: (exact loss, exact gradients, whole-gradient error, per-tensor errors)."""
    loss_fn, sd, stream, out_key, exp = _case(name)
    l0, _, whole, per, g0 = E.grad_errors(loss_fn, sd, stream, out_key, exp)
    return l0, g0, whole, per


def _rel_whole(grads, ref):
    num = sum(float((grads[k].double() - ref[k].double()).pow(2).sum()) for k in ref)
    den = sum(float(ref[k].double().pow(2).sum()) for k in ref)
    return math.sqrt(num / den)


# ------------------------------------------------------------------------------------------------ native steps
class _Batch:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _replay(seq):
    q = list(seq)

    def pop(*a, **k):
        return q.pop(0).clone()
    return pop, q


def _native_denoiser(c, dev):
    """Denoiser.forward + loss.backward() on the native path, the case's draws replayed."""
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig

    inner = c["inner"]
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths),
                                                   inner.num_actions), 0.5, 0.3))
    den.inner_model.load_state_dict(O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"]))
    den = den.to(dev).train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    obs, act, mask, draws = TC.denoiser_inputs(c)
    pop, q = _replay([t.to(dev) for d in draws for t in d])
    o1, o2 = torch.randn, torch.randn_like
    torch.randn, torch.randn_like = pop, pop
    try:
        loss, _ = den(_Batch(obs=obs.to(dev), act=act.to(dev), mask_padding=mask.to(dev)))
    finally:
        torch.randn, torch.randn_like = o1, o2
    assert not q, "Denoiser.forward consumed a different number of random draws"
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {k: p.grad.detach().cpu() for k, p in den.inner_model.named_parameters()}


def _native_rew_end(c, dev):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig

    cfg = c["cfg"]
    m = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                      list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
    m.load_state_dict(O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"]))
    m = m.to(dev).train()
    obs, act, rew, end, mask, final_obs = TC.rew_end_inputs(c)
    info = [{"final_observation": final_obs[i].to(dev)} if i in final_obs else {} for i in range(obs.size(0))]
    batch = _Batch(obs=obs.to(dev).clone(), act=act.to(dev), rew=rew.to(dev), end=end.to(dev), trunc=torch.zeros_like(end).to(dev),
                   mask_padding=mask.to(dev), info=info)
    loss, _ = m(batch)
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {k: p.grad.detach().cpu() for k, p in m.named_parameters()}


class _ScriptedEnv:
    """Returns pre-generated observations / rewards / flags and ignores the action (tests/test_gpu_training.py)."""

    def __init__(self, obs_seq, rew, end, trunc, final_obs, num_actions):
        self.obs_seq, self.rew, self.end, self.trunc, self.final_obs = obs_seq, rew, end, trunc, final_obs
        self.num_envs, self.num_actions, self.t = obs_seq.size(1), num_actions, 0

    def reset(self, seed=None):
        self.t = 0
        return self.obs_seq[0], {}

    def step(self, act):
        t = self.t
        dead = torch.logical_or(self.end[t].bool(), self.trunc[t].bool())
        info = {"final_observation": self.final_obs[t]} if bool(dead.any()) else {}
        self.t += 1
        return self.obs_seq[t + 1], self.rew[t], self.end[t], self.trunc[t], info


def _native_actor_critic(c, dev):
    """ActorCritic.forward (the imagined-rollout loss over the scripted env) + loss.backward(), actions replayed."""
    from torch.distributions.categorical import Categorical

    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig, ActorCriticLossConfig

    cfg = c["cfg"]
    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    ac.load_state_dict(O.seeded_actor_critic_state_dict(cfg, c["wseed"]))
    ac = ac.to(dev).train()
    obs_seq, rew, end, trunc, final_obs, act = TC.actor_critic_inputs(c)
    env = _ScriptedEnv(obs_seq.to(dev), rew.to(dev), end.to(dev), trunc.to(dev), {t: f.to(dev) for t, f in final_obs.items()},
                       cfg.num_actions)
    lc = O.ActorCriticLossCfg(backup_every=c["T"])
    ac.setup_training(env, ActorCriticLossConfig(lc.backup_every, lc.gamma, lc.lambda_, lc.weight_value_loss, lc.weight_entropy_loss))
    acts, step = act.to(dev), [0]

    def replay_sample(self, sample_shape=torch.Size()):
        step[0] += 1
        return acts[:, step[0] - 1]

    orig = Categorical.sample
    Categorical.sample = replay_sample
    try:
        loss, _ = ac()
    finally:
        Categorical.sample = orig
    assert step[0] == c["T"]
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {k: p.grad.detach().cpu() for k, p in ac.named_parameters()}


def _native(name, dev):
    if name in TC.DENOISER_CASES:
        return _native_denoiser(TC.DENOISER_CASES[name], dev)
    if name in TC.REW_END_CASES:
        return _native_rew_end(TC.REW_END_CASES[name], dev)
    return _native_actor_critic(TC.ACTOR_CRITIC_CASES[name], dev)


def _check_case(name, dev):
    loss, grads = _native(name, dev)
    _, again = _native(name, dev)
    _threads()
    ref_loss, ref, emu_whole, emu_per = _budget(name)
    assert set(grads) >= set(ref)
    bad = [k for k, g in grads.items() if not torch.isfinite(g).all()]
    assert not bad, bad[:5]
    flat, flat2 = (torch.cat([d[k].flatten() for k in sorted(d)]).double() for d in (grads, again))
    noise = float((flat2 - flat).norm() / flat.norm())
    e_loss = abs(loss - ref_loss) / abs(ref_loss)
    whole = _rel_whole(grads, ref)
    total = math.sqrt(sum(float(g.pow(2).sum()) for g in ref.values()))
    bound = WHOLE_MARGIN * emu_whole
    rows = []
    for k, r in ref.items():
        e = float((grads[k].double() - r).norm() / r.norm().clamp_min(1e-30))
        rows.append((e, k, float(r.norm()), TENSOR_MARGIN * emu_per[k]))
    worst = max(rows)
    print(f"{name}: loss native {loss:.6f} float64 {ref_loss:.6f} (rel {e_loss:.2e}); whole gradient {whole:.3e} "
          f"(emulation {emu_whole:.3e}, bound {bound:.3e}); worst tensor {worst[1]} {worst[0]:.3e} (bound {worst[3]:.3e}); "
          f"run-to-run {noise:.2e} (bound {RUN_TO_RUN_SHARE * emu_whole:.2e})")
    for e, k, n, tb in sorted(rows, reverse=True)[:5]:
        print(f"   {e:9.3e}  bound {tb:9.3e}  |g|={n:9.3e}  {k}")
    assert bound <= WHOLE_CAP, (name, bound)
    assert e_loss <= 2e-3, (loss, ref_loss)
    assert whole < bound, (whole, bound)
    for e, k, n, tb in rows:
        assert e <= tb or e * n < 1e-4 * total, (k, e, tb, n, total)
        assert e < PER_TENSOR_CAP, (k, e)
    assert noise < RUN_TO_RUN_SHARE * emu_whole, (noise, emu_whole)


ALL_CASES = list(TC.DENOISER_CASES) + list(TC.REW_END_CASES) + list(TC.ACTOR_CRITIC_CASES)


@gpu
@pytest.mark.parametrize("name", ALL_CASES)
def test_training_config_matches_float64_oracle(name):
    _check_case(name, _dev())


# ------------------------------------------------------------------------------------------------ rejections
def _conv_in_denoiser(img_channels, nsc, dev):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig

    inner = O.InnerCfg(img_channels=img_channels, num_steps_conditioning=nsc, cond_channels=224, depths=[1, 1],
                       channels=[32, 32], attn_depths=[0, 0], num_actions=3)
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), 670)
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, nsc, inner.cond_channels, list(inner.depths),
                                                   list(inner.channels), list(inner.attn_depths), inner.num_actions), 0.5, 0.3))
    den.inner_model.load_state_dict(sd)
    b, hw = 2, 16   # the mid blocks attend over 8 x 8 tokens
    obs, act, x = O.synthetic_inputs(b, inner, hw, hw, 671)
    return den.to(dev), inner, sd, obs, act, x


@gpu
@pytest.mark.parametrize("img_channels,nsc", [(6, 7), (9, 7), (16, 7)])
def test_unsupported_conv_in_width_is_refused_before_any_launch(img_channels, nsc):
    """(nsc + 1) * img_channels = 48, 72 and 128 conv_in input channels (48, 80, 128 after padding to 16): conv_in takes 16, 32
    or 64 (the operand prep; the wgrad kernel; at 128 the forward computed a model output 95 % off the float64 oracle's).
    The model is refused when its native handle is created, at the first call, with an error naming conv_in and its channel
    count, nothing launched, the same on a retry; a valid model trains after."""
    from diamond_b200 import _lib

    dev = _dev()
    lib = _lib.lib()
    den, inner, _, obs, act, x = _conv_in_denoiser(img_channels, nsc, dev)
    b, hw = x.shape[0], x.shape[-1]
    args = (x.to(dev), torch.zeros(b, device=dev), obs.reshape(b, -1, hw, hw).to(dev), act.to(dev))
    torch.cuda.synchronize()
    before = lib.dmd_launch_count(0)
    with torch.no_grad(), pytest.raises(RuntimeError) as err:
        den.eval().inner_model(*args)
    after = lib.dmd_launch_count(0)
    msg = str(err.value)
    print(f"img_channels {img_channels}, nsc {nsc}: launches {after - before}; {msg}")
    assert after == before
    assert "conv_in" in msg and f"{(nsc + 1) * img_channels} input channels" in msg, msg
    with pytest.raises(RuntimeError, match="conv_in"):   # training: the same refusal
        den.train().inner_model(*args)
    assert lib.dmd_launch_count(0) == after
    _check_case("D5", dev)


# ------------------------------------------------------------------------------------------------ coverage (CPU)
def _three_pass(cout, cin_store):
    """The Walker's rule (api.cu Walker::conv): a split-fp16 conv whose [W_hi | W_hi | W_lo] pack exceeds 120 KB runs as three
    launches."""
    w1 = 9 * (-(-cin_store // 16) * 16) * (-(-cout // 16) * 16) * 2
    return 3 * w1 > 120 * 1024


def _denoiser_features(c):
    inner = c["inner"]
    d, u, mid = O.unet_block_channels(inner)
    f = set()
    blocks = [b for lv in d + u for b in lv]
    for ci, co, _ in [b for lv in d for b in lv] + [(ci, co, a) for lv in u for ci, co, a in lv]:
        if ci != co:
            f.add(f"proj {ci}->{co}")
    if any(ci == 64 and co == 32 for lv in d for ci, co, _ in lv):
        f.add("projection 64->32 in a d block")
    if any(ci == 32 and co == 64 for lv in d for ci, co, _ in lv):
        f.add("projection 32->64 in a d block")
    if max(len(lv) for lv in u) >= 4:
        f.add("depth-3 level (4 up blocks)")
    if any(a and co == 32 for ci, co, a in blocks):
        f.add("attention in d/u blocks at C=32")
    if mid[0][1] == 32:
        f.add("mid at C=32")
    if len(inner.channels) == 1:
        f.add("no Down/Up records")
    if c["h"] != c["w"]:
        f.add("non-square frames")
    n = len(inner.channels) - 1
    th, tw = c["h"] >> n, c["w"] >> n
    if th * tw == 64 and th != tw:
        f.add("64-token attention as a non-square grid")
    if inner.img_channels > 8:
        f.add("output gradient past 8 channels")
    cin = (inner.num_steps_conditioning + 1) * inner.img_channels
    if _three_pass(inner.channels[0], cin):
        f.add("three-pass conv_in in a training forward")
    if inner.cond_channels == 32:
        f.add("smallest FiLM table")
    if c["b"] == 1:
        f.add("batch of one")
    masked = {bi for bi, _ in c["mask_off"]}
    n_c = inner.num_steps_conditioning
    if c["seq"] >= 3 and any(all((bi, n_c + i) in c["mask_off"] for i in range(c["seq"])) for bi in masked):
        f.add("a sample masked on every step of several")
    return f


def _rew_end_features(c):
    cfg = c["cfg"]
    f = set()
    shapes = dict(O.rew_end_shapes(cfg))
    for k, s in shapes.items():
        if k.endswith("proj.weight") and "attn" not in k:
            f.add(f"proj {s[1]}->{s[0]}")
    if any(a for a in cfg.attn_depths):
        f.add("attention block inside a level")
    if any(cfg.channels[i + 1] < cfg.channels[i] for i in range(len(cfg.channels) - 1)):
        f.add("decreasing channels")
    if max(cfg.depths) >= 3:
        f.add("depth 3")
    if cfg.lstm_dim != O.RewEndCfg().lstm_dim:
        f.add("other LSTM / head width")
    if c["death"] is not None and c["pad"] is not None:
        f.add("a death with its final observation and a padded tail")
    return f


def _actor_critic_features(c):
    cfg = c["cfg"]
    f = set()
    for k, s in O.actor_critic_shapes(cfg):
        if k.endswith("skip_projection.weight"):
            f.add(f"skip {s[1]}->{s[0]}")
    if not all(cfg.down):
        f.add("a level without a max-pool")
    if not cfg.down[0]:
        f.add("no max-pool on the first level")
    if dict(O.actor_critic_shapes(cfg))["lstm.weight_ih"][1] == 4096:
        f.add("LSTM input 4096")
    if cfg.lstm_dim != O.ActorCriticCfg().lstm_dim:
        f.add("other lstm_dim")
    return f


def _features(name):
    if name in TC.DENOISER_CASES:
        return _denoiser_features(TC.DENOISER_CASES[name])
    if name in TC.REW_END_CASES:
        return _rew_end_features(TC.REW_END_CASES[name])
    return _actor_critic_features(TC.ACTOR_CRITIC_CASES[name])


CLAIMS = {
    "D1": {"projection 64->32 in a d block", "depth-3 level (4 up blocks)", "attention in d/u blocks at C=32", "mid at C=32"},
    "D2": {"no Down/Up records"},
    "D3": {"non-square frames", "64-token attention as a non-square grid"},
    "D4": {"output gradient past 8 channels", "three-pass conv_in in a training forward", "projection 64->32 in a d block",
           "projection 32->64 in a d block"},
    "D5": {"smallest FiLM table", "batch of one"},
    "D6": {"a sample masked on every step of several"},
    "R1": {"proj 32->64", "attention block inside a level", "a death with its final observation and a padded tail"},
    "R2": {"decreasing channels", "depth 3", "other LSTM / head width", "proj 64->32"},
    "A1": {"a level without a max-pool", "skip 32->64", "skip 64->32", "LSTM input 4096", "other lstm_dim"},
    "A2": {"no max-pool on the first level", "other lstm_dim"},
}


def test_every_case_reaches_what_it_claims():
    """Each case's features, derived from its config by the oracle's shape walkers and the Walker's three-pass rule, include
    what the case claims; together the cases reach every feature claimed, among them eight that the two denoiser training
    fixtures do not reach."""
    assert set(CLAIMS) == set(ALL_CASES)
    reached = set()
    for name in ALL_CASES:
        f = _features(name)
        print(f"{name}: {sorted(f)}")
        assert CLAIMS[name] <= f, (name, CLAIMS[name] - f)
        reached |= f
    assert set().union(*CLAIMS.values()) <= reached
    from oracle.make_golden import CASES, TRAIN_CASES
    fixtures = set()
    for tc in TRAIN_CASES.values():
        c = CASES[tc["case"]]
        fixtures |= _denoiser_features(dict(c, seq=tc["seq"], mask_off=tc["mask_off"], b=tc["b"]))
    new = set().union(*(CLAIMS[n] for n in TC.DENOISER_CASES)) - fixtures
    print("denoiser features the training fixtures do not reach:", sorted(new))
    assert {"no Down/Up records", "non-square frames", "64-token attention as a non-square grid", "output gradient past 8 channels",
            "three-pass conv_in in a training forward", "depth-3 level (4 up blocks)", "batch of one",
            "a sample masked on every step of several"} <= new, new
    # the default net's conv_in (15 -> 64) is one precise launch; D4's (60 -> 64) is three
    assert not _three_pass(64, 15) and _three_pass(64, 60)


# ------------------------------------------------------------------------------------------------ negative controls (CPU)
def _control_error(name, patch):
    """Whole-gradient relative error of the float64 oracle with `patch` (a context manager) in force, against the plain
    float64 oracle, next to the case's bound (WHOLE_MARGIN x the emulation's error)."""
    loss_fn, sd, stream, out_key, exp = _case(name)
    _, _, emu, _, exact = E.grad_errors(loss_fn, sd, stream, out_key, exp)
    params = {k: v.detach().clone().requires_grad_(v.requires_grad) for k, v in sd.items()}
    with patch(params):
        loss_fn(params).backward()
    wrong = {k: (params[k].grad if params[k].grad is not None else torch.zeros_like(params[k])) for k in exact}
    return _rel_whole(wrong, exact), WHOLE_MARGIN * emu


class _conv_patch:
    """Replaces F.conv2d (which the oracle calls through the module attribute) by f(conv, x, w, b, stride, padding, name)."""

    def __init__(self, f):
        self.f = f

    def __call__(self, params):
        self.names = {id(v): k for k, v in params.items()}
        return self

    def __enter__(self):
        real = F.conv2d

        def conv2d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
            return self.f(real, x, w, b, stride, padding, self.names.get(id(w)))
        self.real, F.conv2d = real, conv2d

    def __exit__(self, *a):
        F.conv2d = self.real


class _skip_detached:
    """One to_cat entry (a skip into an up block) detached: that d-block output's gradient is assigned from its other reader
    instead of accumulated."""

    def __init__(self, prefix, j):
        self.prefix, self.j = prefix, j

    def __call__(self, params):
        return self

    def __enter__(self):
        real = self.real = O.resblocks

        def resblocks(x, cond, sd, p, n, to_cat=None):
            if to_cat is not None and p == self.prefix:
                to_cat = [t.detach() if i == self.j else t for i, t in enumerate(to_cat)]
            return real(x, cond, sd, p, n, to_cat)
        O.resblocks = resblocks

    def __exit__(self, *a):
        O.resblocks = self.real


class _output_channels_zeroed:
    """dL/d(model output) of channels >= 8 dropped: the denoiser backward's 8-channel output gradient."""

    def __call__(self, params):
        return self

    def __enter__(self):
        real = self.real = O.inner_model

        def inner_model(*a, **k):
            y = real(*a, **k)
            if y.requires_grad:
                y.register_hook(lambda g: torch.cat([g[:, :8], torch.zeros_like(g[:, 8:])], 1))
            return y
        O.inner_model = inner_model

    def __exit__(self, *a):
        O.inner_model = self.real


def _second_source_dropped(key, c0):
    """The projection `key` over cat(x, skip) passes no gradient to its second source (channels >= c0)."""
    def f(conv, x, w, b, stride, padding, name):
        if name == key:
            x = torch.cat([x[:, :c0], x[:, c0:].detach()], 1)
        return conv(x, w, b, stride=stride, padding=padding)
    return _conv_patch(f)


def _input_detached(key):
    """The conv `key` passes no gradient to its input (an actor-critic skip projection whose dgrad is not added)."""
    def f(conv, x, w, b, stride, padding, name):
        return conv(x.detach() if name == key else x, w, b, stride=stride, padding=padding)
    return _conv_patch(f)


# D1's u blocks (module order: level 3 .. 0); u_blocks.1 is level 2 (32 channels, skips of 32 then the level's x_down of 64)
CONTROLS = {
    "skip assigned instead of accumulated (D1)": ("D1", lambda: _skip_detached("unet.u_blocks.1.", 1)),
    "second concat source's projection gradient dropped (D1)": ("D1", lambda: _second_source_dropped("unet.u_blocks.1.resblocks.2.proj.weight", 32)),
    "output-gradient channels >= 8 zeroed (D4)": ("D4", _output_channels_zeroed),
    "actor-critic skip projection's gradient not added (A1)": ("A1", lambda: _input_detached("encoder.encoder.3.skip_projection.weight")),
}


@pytest.mark.parametrize("label", list(CONTROLS))
def test_plan_mistakes_miss_the_bound_by_10x(label):
    _threads()
    name, make = CONTROLS[label]
    err, bound = _control_error(name, make())
    print(f"{label}: whole-gradient error {err:.3e}, bound {bound:.3e}, ratio {err / bound:.0f}x")
    assert err >= CONTROL_MARGIN * bound, (err, bound)


def test_control_targets_exist():
    """The controls name layers that exist where they are applied: D1's u_blocks.1.resblocks.2 projects cat(32, 64) -> 64,
    A1's level without a max-pool has a 32 -> 64 skip projection, D4 has 12 output channels."""
    d1 = dict(O.inner_model_shapes(TC.DENOISER_CASES["D1"]["inner"]))
    assert d1["unet.u_blocks.1.resblocks.2.proj.weight"] == (64, 96, 1, 1)
    assert len([k for k in d1 if k.startswith("unet.u_blocks.1.") and k.endswith("conv1.weight")]) == 3
    a1 = dict(O.actor_critic_shapes(TC.ACTOR_CRITIC_CASES["A1"]["cfg"]))
    assert a1["encoder.encoder.3.skip_projection.weight"] == (64, 32, 1, 1)
    assert TC.DENOISER_CASES["D4"]["inner"].img_channels == 12


# ------------------------------------------------------------------------------------------------ oracle vs reference (CPU)
@pytest.mark.parametrize("name", TC.GOLDEN_CASES)
def test_float64_oracle_matches_reference_at_new_configs(golden_dir, name):
    """The float64 checker's loss and gradients at D1 / D4 against the unmodified reference's (fp32) run on the same inputs
    (tests/golden/training_config_<id>.npz, oracle/training_configs.py)."""
    _threads()
    g = np.load(os.path.join(golden_dir, f"training_config_{name.lower()}.npz"))
    c = TC.DENOISER_CASES[name]
    obs, act, mask, draws = TC.denoiser_inputs(c)
    assert abs(TC.inputs_checksum([obs, act, mask] + [t for s in draws for t in s]) - float(g["inputs_checksum"])) < 1e-9 * float(g["inputs_checksum"])
    sd = _denoiser_sd(c)
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    loss = _denoiser_loss_fn(c)(sd)
    print(f"{name}: loss float64 {loss.item():.8f} reference {float(g['loss']):.8f}")
    assert abs(loss.item() - float(g["loss"])) <= 2e-5 * abs(float(g["loss"]))
    loss.backward()
    named = [(k, v.grad) for k, v in sd.items() if k != "noise_emb.weight"]
    keys, norms, samples = O.grad_summary(named)
    assert keys == [str(k) for k in g["grad_keys"]]
    ref_n, ref_s = g["grad_norms"], g["grad_samples"]
    total = float(np.sqrt((ref_n ** 2).sum()))
    assert np.all(np.abs(norms - ref_n) <= 2e-4 * ref_n + 1e-6 * total), float(np.max(np.abs(norms - ref_n) / (ref_n + 1e-12)))
    numel = np.array([gr.numel() for _, gr in named], np.float64)
    scale = (ref_n / np.sqrt(numel))[:, None]
    assert np.all(np.abs(samples - ref_s) <= 2e-4 * np.abs(ref_s) + 2e-3 * scale + 1e-9)
