"""Cost of smaller frames on the default nets (denoiser [64] * 4 with depths 2, reward / termination [32] * 4, actor-critic
[32, 32, 64, 64] with four max-pools, frame stack 4, RGB).  Per frame size S in {32, 40, 48, 56, 64}, with CUDA events after a
warm-up:

* `sample_ms`: DiffusionSampler.sample() at 32 envs and 3 Euler steps (device-resident, CUDA graph);
* `train_ms`: the cfg-2 step of bench.py at batch 256 (Denoiser.forward + backward + clip_grad_norm_ + AdamW, one
  autoregressive step);
* `rew_end_ms`: the reward / termination step at 32 segments x 19 frames (RewEndModel.forward + backward + clip + AdamW);
* `ac_update_ms`: the cfg-3 update of bench.py (32 envs x horizon 15 in imagination, 3 denoising steps, + BPTT + clip + AdamW).

Then, in a run of its own, a torch.profiler trace of one cfg-2 step gives the share of the step's kernel time taken by
gn_stats_kernel, which supplies the GroupNorm statistics of convs on levels below 7 x 7 (the conv's statistics epilogue keeps
three images per tile).  At S = 64 the launches per sample() and per training step are counted and the sample()
output is hashed, so that two trees can be compared.  The card, its power limit and SM clocks are read in the same run.

Comparing two source trees (this one and a parent, each with its native library built) runs the worker for each tree in fresh
processes, alternating the order round by round; a size a tree refuses is reported as refused:

    python scripts/bench_small_frames.py --trees . ../parent --rounds 2 --out result.json
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMED = ("sample_ms", "train_ms", "rew_end_ms", "ac_update_ms")


def _card():
    import torch

    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out["power_limit_sm_clock_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand; the card's limits are then unknown
        out["power_limit_sm_clock_max_sm_clock"] = f"unknown ({e})"
    return out


def _timed(fn, warmup, steps):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _launches(fn):
    import torch

    from diamond_b200 import _lib

    torch.cuda.synchronize()
    _lib.lib().dmd_launch_count(1)
    fn()
    torch.cuda.synchronize()
    return int(_lib.lib().dmd_launch_count(0))


def _denoiser(a, S, r, dev):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from diamond_b200.models.diffusion import (Denoiser, DenoiserConfig, DiffusionSampler, DiffusionSamplerConfig,
                                               InnerModelConfig, SigmaDistributionConfig)
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0, 0, 0, 0], 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    den = den.to(dev).eval()
    obs, act, _ = frame_stacks(a.envs, 4, 3, S, S, 4, 100)
    obs, act = obs.to(dev), act.to(dev)
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(3))
    r["sample_ms"] = _timed(lambda: sampler.sample(obs, act), a.warmup, a.steps)
    if S == 64:
        r["sample_launches"] = _launches(lambda: sampler.sample(obs, act))
        torch.manual_seed(5)
        x, _ = sampler.sample(obs, act)
        r["sample_sha256"] = hashlib.sha256(x.cpu().numpy().tobytes()).hexdigest()

    den.train()
    den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
    opt = torch.optim.AdamW(den.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    tobs, tact, _ = frame_stacks(a.batch, 5, 3, S, S, 4, 300)
    b = types.SimpleNamespace(obs=tobs.to(dev), act=tact.to(dev), mask_padding=torch.ones(a.batch, 5, dtype=torch.bool, device=dev))

    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = den(b)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(den.parameters(), 1.0)
        opt.step()
    r["train_ms"] = _timed(step, a.warmup, a.steps)
    if S == 64:
        r["train_launches"] = _launches(step)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:   # in a run of its own, after the timed steps
        step()
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type.name == "CUDA"]
    total_us = sum(e.device_time for e in kern)
    stats = [e.device_time for e in kern if "gn_stats_kernel" in e.name]
    r["train_profile_kernel_ms"] = total_us / 1e3
    r["train_gn_stats"] = {"launches": len(stats), "us": sum(stats), "share_of_step_kernel_time": sum(stats) / total_us if total_us else None}


def _rew_end(a, S, r, dev):
    import numpy as np
    import torch

    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import randomize_module_
    from oracle import rew_end_training as RT
    from oracle import torch_oracle as O

    c = O.RewEndCfg(img_size=S)
    m = RewEndModel(RewEndModelConfig(c.lstm_dim, c.img_channels, c.img_size, c.cond_channels, list(c.depths), list(c.channels),
                                      list(c.attn_depths), c.num_actions))
    randomize_module_(m, 7)
    m = m.to(dev).train()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    rng = np.random.default_rng(1901)
    n, T = 32, 19
    obs = RT.frames(rng.integers(0, 256, size=(n, T, c.img_channels, S, S), dtype=np.uint8)).to(dev)
    act = torch.from_numpy(rng.integers(0, c.num_actions, size=(n, T))).to(dev)
    rew = torch.from_numpy(rng.choice([-1.0, 0.0, 0.0, 1.0], size=(n, T)).astype(np.float32)).to(dev)
    end = torch.zeros(n, T, dtype=torch.long, device=dev)
    mask = torch.ones(n, T, dtype=torch.bool, device=dev)
    end[1, 9] = 1
    mask[1, 10:] = False
    info = [{"final_observation": obs[1, 10].clone()} if i == 1 else {} for i in range(n)]

    def step():
        b = types.SimpleNamespace(obs=obs.clone(), act=act, rew=rew, end=end, trunc=torch.zeros_like(end), mask_padding=mask, info=info)
        opt.zero_grad(set_to_none=True)
        loss, _ = m(b)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(m.parameters(), 100.0)
        opt.step()
    r["rew_end_ms"] = _timed(step, a.warmup, a.steps)


def _ac_update(a, S, r, dev, horizon=15):
    """bench.py's imagination_block at frame size S, one process, no all-reduce."""
    import torch

    from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig, ActorCriticLossConfig
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, DiffusionSamplerConfig, InnerModelConfig
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    rem = RewEndModel(RewEndModelConfig(512, 3, S, 128, [2, 2, 2, 2], [32] * 4, [0] * 4, 4))
    randomize_module_(rem, 2025)
    ac = ActorCritic(ActorCriticConfig(512, 3, S, [32, 32, 64, 64], [1, 1, 1, 1], 4))
    randomize_module_(ac, 2026)
    den, rem, ac = den.to(dev).eval(), rem.to(dev).eval(), ac.to(dev).train()
    with torch.no_grad():   # rare episode ends, as bench.py
        last = [m for m in rem.modules() if isinstance(m, torch.nn.Linear)][-1]
        last.weight[3].fill_(0.05); last.weight[4].fill_(-0.05)
    envs = a.envs
    pool = [frame_stacks(envs, 4, 3, S, S, 4, 1000 + k)[:2] for k in range(8)]

    class Loader:
        batch_sampler = types.SimpleNamespace(batch_size=envs)

        def __iter__(self):
            k = 0
            while True:
                obs, act = pool[k % len(pool)]
                k += 1
                yield types.SimpleNamespace(obs=obs, act=act)

    env = WorldModelEnv(den, rem, Loader(), WorldModelEnvConfig(horizon, 4, DiffusionSamplerConfig(3)))
    ac.setup_training(env, ActorCriticLossConfig(horizon, 0.985, 0.95, 1.0, 0.001))
    opt = torch.optim.AdamW(ac.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)

    def update():
        opt.zero_grad(set_to_none=True)
        loss, _ = ac()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(ac.parameters(), 100.0)
        opt.step()
    r["ac_update_ms"] = _timed(update, 1, max(1, a.steps // 3))


def worker(a):
    import torch

    sys.path.insert(0, os.getcwd())
    dev = torch.device("cuda:0")
    out = {"card": _card(), "sizes": {}}
    for S in a.sizes:
        r = {}
        for part in (_denoiser, _rew_end, _ac_update):
            try:
                part(a, S, r, dev)
            except Exception as e:   # a tree that refuses this size
                r.setdefault("refused", {})[part.__name__.strip("_")] = str(e).splitlines()[0][:200]
            torch.cuda.empty_cache()
        out["sizes"][str(S)] = r
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=["."], help="source trees whose diamond_b200 package is measured")
    ap.add_argument("--sizes", type=int, nargs="+", default=[32, 40, 48, 56, 64])
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--envs", type=int, default=32)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    runs = {t: [] for t in a.trees}
    for rnd in range(a.rounds):
        for t in (a.trees if rnd % 2 == 0 else a.trees[::-1]):
            env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.abspath(t), ROOT]))
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--steps", str(a.steps), "--warmup", str(a.warmup),
                   "--envs", str(a.envs), "--batch", str(a.batch), "--sizes", *map(str, a.sizes)]
            res = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=os.path.abspath(t))
            if res.returncode != 0:
                raise SystemExit(f"{t}: worker failed\n{res.stdout}\n{res.stderr}")
            runs[t].append(json.loads(res.stdout.strip().splitlines()[-1]))
            print(t, "round", rnd, json.dumps(runs[t][-1]), flush=True)
    summary = {"rounds": a.rounds, "steps": a.steps, "warmup": a.warmup, "trees": {}}
    for t, rs in runs.items():
        summary["card"] = rs[-1]["card"]
        tree = summary["trees"][t] = {}
        for S in map(str, a.sizes):
            per = [x["sizes"][S] for x in rs]
            keys = [k for k in TIMED if all(k in p for p in per)]
            tree[S] = dict(per[-1], **{k: statistics.median(p[k] for p in per) for k in keys},
                           **{k + "_all": [p[k] for p in per] for k in keys})
    print(json.dumps(summary))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
