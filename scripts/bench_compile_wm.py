"""The cfg-3 imagination update (bench.py's imagination_block: ActorCritic.forward() over WorldModelEnv at 32 envs x horizon
15, 3 denoising steps, then backward, clip and AdamW) with the reference trainer's `training.compile_wm` off and on
(torch.compile(..., mode="reduce-overhead") of predict_next_obs and predict_rew_end, trainer.py:182-184).

The two settings alternate in one process; each is timed over `--updates` updates per round, and the median of `--rounds`
rounds is reported.  Also reported: the first compiled update (compile, warm-up and CUDA-graph recording), predict_rew_end
per call, and the native kernels the host launches per imagined step (dmd_launch_count; 0 when the step replays the
recorded graphs).  Prints one JSON line with the card's name and power limit.

    python scripts/bench_compile_wm.py [--rounds 3] [--updates 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        limit = f"unknown ({e!r})"
    return name, limit


def world(dev, compiled, envs=32, horizon=15):
    import torch

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
    with torch.no_grad():   # P(end) of a few per cent, as in bench.py
        last = [m for m in rem.modules() if isinstance(m, torch.nn.Linear)][-1]
        last.weight[3].fill_(0.05); last.weight[4].fill_(-0.05)
    pool = [frame_stacks(envs, 4, 3, 64, 64, 4, 1000 + k)[:2] for k in range(8)]

    class Loader:
        batch_sampler = types.SimpleNamespace(batch_size=envs)

        def __iter__(self):
            k = 0
            while True:
                obs, act = pool[k % len(pool)]
                k += 1
                yield types.SimpleNamespace(obs=obs, act=act)

    env = WorldModelEnv(den, rem, Loader(), WorldModelEnvConfig(horizon, 4, DiffusionSamplerConfig(3)))
    if compiled:
        env.predict_next_obs = torch.compile(env.predict_next_obs, mode="reduce-overhead")
        env.predict_rew_end = torch.compile(env.predict_rew_end, mode="reduce-overhead")
    ac.setup_training(env, ActorCriticLossConfig(horizon, 0.985, 0.95, 1.0, 0.001))
    opt = torch.optim.AdamW(ac.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    return env, ac, opt


def update(ac, opt):
    import torch

    opt.zero_grad(set_to_none=True)
    loss, _ = ac()
    loss.backward()
    torch.nn.utils.clip_grad_norm_(ac.parameters(), 100.0)
    opt.step()


def time_updates(ac, opt, n):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        update(ac, opt)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def rew_end_ms(env, calls=200):
    """predict_rew_end alone, on the ring as env.step leaves it (head fixed: one graph)."""
    import torch

    nxt = env._frames[env._head].unsqueeze(1)
    for _ in range(3):
        env.predict_rew_end(nxt)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        env.predict_rew_end(nxt)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / calls


def launches_per_step(env, steps=8):
    """Native kernels the host launches per imagined step without deaths (predict_next_obs + predict_rew_end)."""
    import torch

    from diamond_b200 import _lib

    lib, t = _lib.lib(), env._frames.size(0)

    def run(n):
        for _ in range(n):
            nxt, _ = env.predict_next_obs()
            env.predict_rew_end(nxt.unsqueeze(1))
            env._head = (env._head + 1) % t
    run(2 * t)   # every ring head once more in this call pattern
    torch.cuda.synchronize()
    n0 = lib.dmd_launch_count(0)
    run(steps)
    torch.cuda.synchronize()
    return (lib.dmd_launch_count(0) - n0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates", type=int, default=3)
    a = ap.parse_args()
    import torch

    dev = torch.device("cuda:0")
    name, limit = card()
    worlds = {}
    t0 = time.perf_counter()
    worlds[False] = world(dev, False)
    update(*worlds[False][1:])                     # eager warm-up: handles, packs, the sampler's own graphs
    torch.cuda.synchronize()
    eager_first_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    worlds[True] = world(dev, True)
    update(*worlds[True][1:])                      # compile, warm-up and recording of every ring head
    torch.cuda.synchronize()
    compiled_first_ms = (time.perf_counter() - t0) * 1e3
    update(*worlds[True][1:])
    rounds = {False: [], True: []}
    for _ in range(a.rounds):
        for compiled in (False, True):
            rounds[compiled].append(time_updates(*worlds[compiled][1:], a.updates))
    out = {
        "card": name, "power_limit": limit,
        "update_ms_eager": statistics.median(rounds[False]), "update_ms_compiled": statistics.median(rounds[True]),
        "rounds_eager": rounds[False], "rounds_compiled": rounds[True],
        "first_update_ms_eager": eager_first_ms, "first_update_ms_compiled": compiled_first_ms,
        "native_launches_per_step_eager": launches_per_step(worlds[False][0]),
        "native_launches_per_step_compiled": launches_per_step(worlds[True][0]),
        "predict_rew_end_ms_eager": rew_end_ms(worlds[False][0]), "predict_rew_end_ms_compiled": rew_end_ms(worlds[True][0]),
        "updates_per_round": a.updates, "envs": 32, "horizon": 15,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
