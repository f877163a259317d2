"""Cost of deterministic mode (torch.use_deterministic_algorithms(True)) on the default nets, flag off and on in alternating
rounds in one process, CUDA events after a warm-up of each shape in each mode:

* `sample_ms`: DiffusionSampler.sample() at 32 envs and 3 Euler steps (device-resident, CUDA graph);
* `train_ms`: the cfg-2 step of bench.py at batch 256 (Denoiser.forward + backward + clip_grad_norm_ + AdamW);
* `rew_end_ms`: the reward / termination step at 32 segments x 19 frames (RewEndModel.forward + backward + clip + AdamW);
* `imagination_ms`: the cfg-3 update of bench.py (`imagination_block`: ActorCritic.forward() over WorldModelEnv at 32 envs x
  horizon 15 with the native sampler and reward / termination model, BPTT backward, clip + AdamW), mean of 3 updates after 1.

The card, its power limit and SM clocks are read in the same run.

    python scripts/bench_deterministic.py --rounds 3 --out result.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

# torch's cuBLAS calls (the optimizer's and torch's own ops) refuse deterministic mode without a fixed workspace configuration
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    import torch

    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out["power_limit_max_sm_clock_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand; the card's limits are then unknown
        out["power_limit_max_sm_clock_sm_clock"] = f"unknown ({e})"
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--envs", type=int, default=32)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import numpy as np
    import torch

    from diamond_b200.models.diffusion import (Denoiser, DenoiserConfig, DiffusionSampler, DiffusionSamplerConfig,
                                               InnerModelConfig, SigmaDistributionConfig)
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_
    from bench import imagination_block
    from oracle import rew_end_training as RT
    from oracle import torch_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic: needs a CUDA device")
    dev = torch.device("cuda:0")

    class B_:
        pass

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0, 0, 0, 0], 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    den = den.to(dev)
    obs, act, _ = frame_stacks(a.envs, 4, 3, 64, 64, 4, 100)
    obs, act = obs.to(dev), act.to(dev)
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(3))
    den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
    opt = torch.optim.AdamW(den.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    tobs, tact, _ = frame_stacks(a.batch, 5, 3, 64, 64, 4, 300)
    tb = B_()
    tb.obs, tb.act, tb.mask_padding = tobs.to(dev), tact.to(dev), torch.ones(a.batch, 5, dtype=torch.bool, device=dev)

    def sample():
        den.eval()
        sampler.sample(obs, act)

    def train():
        den.train()
        opt.zero_grad(set_to_none=True)
        loss, _ = den(tb)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(den.parameters(), 1.0)
        opt.step()

    c = O.RewEndCfg()
    m = RewEndModel(RewEndModelConfig(c.lstm_dim, c.img_channels, c.img_size, c.cond_channels, list(c.depths), list(c.channels),
                                      list(c.attn_depths), c.num_actions))
    randomize_module_(m, 7)
    m = m.to(dev).train()
    ropt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    rng = np.random.default_rng(1901)
    S, T = 32, 19
    robs = RT.frames(rng.integers(0, 256, size=(S, T, c.img_channels, c.img_size, c.img_size), dtype=np.uint8)).to(dev)
    ract = torch.from_numpy(rng.integers(0, c.num_actions, size=(S, T))).to(dev)
    rrew = torch.from_numpy(rng.choice([-1.0, 0.0, 0.0, 1.0], size=(S, T)).astype(np.float32)).to(dev)
    rend = torch.zeros(S, T, dtype=torch.long, device=dev)
    rmask = torch.ones(S, T, dtype=torch.bool, device=dev)
    rend[1, 9] = 1
    rmask[1, 10:] = False
    info = [{"final_observation": robs[1, 10].clone()} if i == 1 else {} for i in range(S)]

    def rew_end():
        rb = B_()
        rb.obs, rb.act, rb.rew, rb.end, rb.mask_padding, rb.info = robs.clone(), ract, rrew, rend, rmask, info
        rb.trunc = torch.zeros_like(rend)
        ropt.zero_grad(set_to_none=True)
        loss, _ = m(rb)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(m.parameters(), 100.0)
        ropt.step()

    out = {"card": _card(), "rounds": []}
    for r in range(a.rounds):
        row = {}
        for mode in ((False, True) if r % 2 == 0 else (True, False)):
            torch.use_deterministic_algorithms(mode)
            key = "on" if mode else "off"
            row[key] = {"sample_ms": _timed(sample, a.warmup, a.steps), "train_ms": _timed(train, a.warmup, a.steps),
                        "rew_end_ms": _timed(rew_end, a.warmup, a.steps),
                        "imagination_ms": imagination_block(dev, 1, 0, envs=a.envs)["ms_per_update"]}
        torch.use_deterministic_algorithms(False)
        out["rounds"].append(row)
        print(json.dumps({"round": r, **row}), flush=True)
    out["median"] = {k: {q: statistics.median(rr[k][q] for rr in out["rounds"]) for q in out["rounds"][0][k]} for k in ("off", "on")}
    out["card_after"] = _card()
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
