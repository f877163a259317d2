"""Cost of a wider conditioning vector: cond_channels in {256, 512, 1024, 2048} on the default levels ([64] * 4, depths 2, 64 x 64
RGB frames, frame stack 4).  Per width, with CUDA events after a warm-up:

* `sample_ms`: DiffusionSampler.sample() at 32 envs and 3 Euler steps (device-resident, CUDA graph);
* `train_ms`: the cfg-2 step of bench.py at batch 256 (Denoiser.forward + backward + clip_grad_norm_ + AdamW, one autoregressive
  step);
* `rew_end_ms`: the reward / termination step at 32 segments x 19 frames (RewEndModel.forward + backward + clip + AdamW).

Then, in a run of its own, a torch.profiler trace of one training step gives the kernel time of the FiLM forward (the batched
FiLM linear: linear_kernel with F = FiLM rows), the FiLM weight gradient (film_wgrad_kernel) and dcond = dfilm Wf (the split-K
sgemm_kernel + splitk_reduce_kernel of film_tail), with FLOP and bytes counted from the shapes, and their share of the step's
kernel time.  The card, its power limit and SM clocks are read in the same run.

Comparing two source trees (this one and a parent, each with its native library built) runs the worker for each tree in fresh
processes, alternating the order round by round; only widths a tree accepts are measured there:

    python scripts/bench_cond_width.py --trees . ../parent --rounds 3 --widths 256 512 1024 2048 --out result.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def film_costs(film_rows, cc, b):
    """(FLOP, bytes) from the shapes of the three FiLM ops at batch b (fp32 operands, each read or written once)."""
    return {
        "film_fwd": (2.0 * b * film_rows * cc, 4.0 * (film_rows * cc + b * cc + b * film_rows + film_rows)),
        "film_wgrad": (2.0 * b * film_rows * (cc + 1), 4.0 * (b * film_rows + b * cc + 2 * (film_rows * cc + film_rows))),
        "dcond": (2.0 * b * film_rows * cc, 4.0 * (b * film_rows + film_rows * cc + b * cc)),
    }


def worker(a):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    sys.path.insert(0, os.getcwd())
    from diamond_b200.models.diffusion import (Denoiser, DenoiserConfig, DiffusionSampler, DiffusionSamplerConfig,
                                               InnerModelConfig, SigmaDistributionConfig)
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    dev = torch.device("cuda:0")
    out = {"card": _card(), "widths": {}}

    class B_:
        pass

    for cc in a.widths:
        r = {}
        try:
            den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, cc, [2, 2, 2, 2], [64] * 4, [0, 0, 0, 0], 4), 0.5, 0.3))
            randomize_module_(den.inner_model, 2024)
            den = den.to(dev).eval()
            den.inner_model.native()
        except Exception as e:   # a tree that refuses this width
            out["widths"][str(cc)] = {"refused": str(e).splitlines()[0][:200]}
            continue
        film_rows = sum(m.linear.weight.shape[0] for m in den.inner_model.modules() if type(m).__name__ == "AdaGroupNorm")
        r["film_rows"] = film_rows
        obs, act, _ = frame_stacks(a.envs, 4, 3, 64, 64, 4, 100)
        obs, act = obs.to(dev), act.to(dev)
        sampler = DiffusionSampler(den, DiffusionSamplerConfig(3))
        r["sample_ms"] = _timed(lambda: sampler.sample(obs, act), a.warmup, a.steps)

        den.train()
        den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
        opt = torch.optim.AdamW(den.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
        tobs, tact, _ = frame_stacks(a.batch, 5, 3, 64, 64, 4, 300)
        b = B_()
        b.obs, b.act, b.mask_padding = tobs.to(dev), tact.to(dev), torch.ones(a.batch, 5, dtype=torch.bool, device=dev)

        def step():
            opt.zero_grad(set_to_none=True)
            loss, _ = den(b)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(den.parameters(), 1.0)
            opt.step()
        r["train_ms"] = _timed(step, a.warmup, a.steps)

        # the profiled step, in a run of its own after the timed ones
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if e.device_type.name == "CUDA"]
        total_us = sum(e.device_time for e in kern)

        def us(pred):
            return sum(e.device_time for e in kern if pred(e.name))
        # linear_kernel runs three times per forward (cond MLP 2x CC -> CC, FiLM CC -> rows) and once more in the backward (the
        # cond MLP's pre-activation recompute); the FiLM one is the largest, K = CC over F = rows > CC outputs
        lin = sorted((e.device_time for e in kern if "linear_kernel" in e.name), reverse=True)
        # dcond: the split-K sgemm_kernel and its splitk_reduce_kernel that follow film_wgrad_kernel (BwdBuilder::film_tail)
        kern.sort(key=lambda e: e.time_range.start)
        i = next((j for j, e in enumerate(kern) if "film_wgrad_kernel" in e.name), len(kern))
        sg = next((e.device_time for e in kern[i:] if "sgemm_kernel" in e.name), 0.0)
        red = next((e.device_time for e in kern[i:] if "splitk_reduce_kernel" in e.name), 0.0)
        ops = {"film_fwd": lin[0] if lin else 0.0, "film_wgrad": us(lambda n: "film_wgrad_kernel" in n), "dcond": sg + red}
        costs = film_costs(film_rows, cc, a.batch)
        r["profile_step_kernel_ms"] = total_us / 1e3
        r["film_ops"] = {k: {"us": v, "share_of_step_kernel_time": v / total_us if total_us else None,
                             "gflop": costs[k][0] / 1e9, "mbytes": costs[k][1] / 1e6,
                             "tflop_per_s": costs[k][0] / (v * 1e-6) / 1e12 if v else None,
                             "gb_per_s": costs[k][1] / (v * 1e-6) / 1e9 if v else None} for k, v in ops.items()}
        del den, opt, sampler, b
        torch.cuda.empty_cache()

        from oracle import rew_end_training as RT
        from oracle import torch_oracle as O

        c = O.RewEndCfg(cond_channels=cc)
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

        def rstep():
            rb = B_()
            rb.obs, rb.act, rb.rew, rb.end, rb.mask_padding, rb.info = robs.clone(), ract, rrew, rend, rmask, info
            rb.trunc = torch.zeros_like(rend)
            ropt.zero_grad(set_to_none=True)
            loss, _ = m(rb)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(m.parameters(), 100.0)
            ropt.step()
        r["rew_end_ms"] = _timed(rstep, a.warmup, a.steps)
        del m, ropt
        torch.cuda.empty_cache()
        out["widths"][str(cc)] = r
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=["."], help="source trees whose diamond_b200 package is measured")
    ap.add_argument("--widths", type=int, nargs="+", default=[256, 512, 1024, 2048])
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
    for r in range(a.rounds):
        for t in (a.trees if r % 2 == 0 else a.trees[::-1]):
            env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.abspath(t), ROOT]))
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--steps", str(a.steps), "--warmup", str(a.warmup),
                   "--envs", str(a.envs), "--batch", str(a.batch), "--widths", *map(str, a.widths)]
            res = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=os.path.abspath(t))
            if res.returncode != 0:
                raise SystemExit(f"{t}: worker failed\n{res.stdout}\n{res.stderr}")
            runs[t].append(json.loads(res.stdout.strip().splitlines()[-1]))
            print(t, "round", r, json.dumps(runs[t][-1]), flush=True)
    summary = {"rounds": a.rounds, "steps": a.steps, "warmup": a.warmup, "trees": {}}
    for t, rs in runs.items():
        summary["card"] = rs[-1]["card"]
        tree = summary["trees"][t] = {}
        for cc in map(str, a.widths):
            per = [x["widths"][cc] for x in rs]
            if "refused" in per[-1]:
                tree[cc] = per[-1]
                continue
            tree[cc] = dict(per[-1], **{k: statistics.median(p[k] for p in per) for k in ("sample_ms", "train_ms", "rew_end_ms")},
                            **{k + "_all": [p[k] for p in per] for k in ("sample_ms", "train_ms", "rew_end_ms")})
    print(json.dumps(summary))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
