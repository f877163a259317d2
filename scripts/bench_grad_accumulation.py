"""Optimizer steps of the denoiser (cfg 2 of BASELINE.json: 64 channels x 4 levels, cond 256, 64 x 64 frames) that run more
than one native backward node before AdamW, with the gradients accumulated natively into one flat buffer or not:

* `ar2`: batch 256, num_autoregressive_steps = 2 (two nodes in one backward pass);
* `acc2`: grad_acc_steps = 2 at micro-batch 128, one autoregressive step (two backward passes, no zero_grad between them).

Per workload: ms per optimizer step (forward + backward passes + clip_grad_norm_ + AdamW, CUDA events, after warm-up), the
memory the step allocates above what is allocated before it (torch.cuda.max_memory_allocated), the kernels launched during
the last backward pass and how many of them are torch's (autograd's per-tensor gradient adds; torch.profiler, one step of its
own), the distinct buffers the `.grad`s live in, whether they alias `last_flat_grad` (allreduce_native_gradients then reduces
that buffer in place; otherwise it copies into buckets and back), and the collectives it would issue on more than one rank.

Comparing two source trees (e.g. this commit and its parent, each with its native library built) alternates them round by
round in fresh processes, so both see the same GPU state:

    python scripts/bench_grad_accumulation.py --trees . ../parent --rounds 3 --steps 10 --warmup 3 --out result.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

WORKLOADS = {"ar2": dict(micro=256, passes=1, ar_steps=2), "acc2": dict(micro=128, passes=2, ar_steps=1)}


def _buckets(numels, bucket_bytes=32 << 20):
    """The collectives utils.allreduce_gradients issues for parameters of these sizes (its greedy bucketing)."""
    calls, i = 0, 0
    while i < len(numels):
        j, nbytes = i, 0
        while j < len(numels) and (j == i or nbytes + numels[j] * 4 <= bucket_bytes):
            nbytes += numels[j] * 4
            j += 1
        calls, i = calls + 1, j
    return calls


def worker(args):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(0)}
    for name, w in WORKLOADS.items():
        den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
        randomize_module_(den.inner_model, 2024)
        den = den.to(dev).train()
        den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
        params = list(den.parameters())
        opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=1e-2, eps=1e-8)
        T = 4 + w["ar_steps"]
        batches = []
        for k in range(w["passes"]):
            obs, act, _ = frame_stacks(w["micro"], T, 3, 64, 64, 4, 300 + k)

            class B_:
                pass
            b = B_()
            b.obs, b.act, b.mask_padding = obs.to(dev), act.to(dev), torch.ones(w["micro"], T, dtype=torch.bool, device=dev)
            batches.append(b)

        def step(prof=None):
            opt.zero_grad(set_to_none=True)
            for k, b in enumerate(batches):
                loss, _ = den(b)
                if prof is not None and k == len(batches) - 1:
                    with prof:
                        loss.backward()
                        torch.cuda.synchronize()
                else:
                    loss.backward()
            torch.nn.utils.clip_grad_norm_(params, 1.0)
            opt.step()

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.steps):
            step()
        ev[1].record()
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / args.steps
        opt.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step()
        torch.cuda.synchronize()
        peak_mb = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        storages = {p.grad.untyped_storage().data_ptr() for p in params}
        flat = getattr(den.inner_model, "last_flat_grad", None)
        aliased = flat is not None and storages == {flat.untyped_storage().data_ptr()}
        prof = profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA])
        step(prof)
        torch.cuda.synchronize()
        kernels = [e.name for e in prof.events() if e.device_type.name == "CUDA" and "mem" not in e.name.lower()]
        torch_kernels = sum(1 for k in kernels if "at::" in k)   # torch's own kernels (the native library's are not in at::)
        out[name] = {"ms_per_step": ms, "step_alloc_peak_mb": peak_mb, "last_backward_kernels": len(kernels),
                     "last_backward_torch_kernels": torch_kernels,
                     "grad_buffers": len(storages),
                     "grads_alias_last_flat_grad": aliased,
                     "collectives_per_step": 1 if aliased else _buckets([p.numel() for p in params]),
                     "flat_grad_mb": den.inner_model._grad_views_layout()[2] * 4 / 2 ** 20}
        del den, opt, batches, params
        torch.cuda.empty_cache()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=["."], help="source trees whose diamond_b200 package is measured")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    runs = {t: [] for t in args.trees}
    for r in range(args.rounds):
        for t in (args.trees if r % 2 == 0 else args.trees[::-1]):
            env = dict(os.environ, PYTHONPATH=os.path.abspath(t))
            res = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--steps", str(args.steps), "--warmup",
                                  str(args.warmup)], env=env, capture_output=True, text=True, cwd=os.path.abspath(t))
            if res.returncode != 0:
                raise SystemExit(f"{t}: worker failed\n{res.stdout}\n{res.stderr}")
            runs[t].append(json.loads(res.stdout.strip().splitlines()[-1]))
            print(t, "round", r, json.dumps(runs[t][-1]), flush=True)
    summary = {"gpu": gpu, "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup, "trees": {}}
    for t, rs in runs.items():
        summary["trees"][t] = {}
        for name in WORKLOADS:
            per = [r[name] for r in rs]
            ms = [p["ms_per_step"] for p in per]
            summary["trees"][t][name] = dict(per[-1], ms_per_step=statistics.median(ms), ms_per_step_all=ms)
    print(json.dumps(summary))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
