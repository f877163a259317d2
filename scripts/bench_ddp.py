"""Training steps of the native models wrapped in torch DistributedDataParallel (`DDP(module)` with its default arguments, as
the reference trainer wraps them, utils.py:105-106) against the same step without the wrapper:

* `cfg2`: the denoiser step of BASELINE.json cfg 2 (batch 256 per GPU, 1 autoregressive step, clip + AdamW);
* `cfg3`: the actor-critic update of cfg 3 (32 environments x horizon 15 through WorldModelEnv, clip + AdamW).

Modes, alternated round by round on the same GPU (each mode has its own model, built from the same seeds):

* `direct`: the model called without a wrapper, followed by `allreduce_native_gradients` (ONE all-reduce of the flat gradient
  buffer; at world 1 it issues nothing, so this is the step without any process group work);
* `ddp`: the model called through DDP, whose hooks average the gradients in buckets.

Per workload and mode: the median over rounds of ms per step (CUDA events around `--steps` steps after `--warmup`, MAX over
ranks).  Then, outside the timed steps: how many times the native weights are re-packed in one step, and in a second forward
without an optimizer step between (grad_acc_steps = 2), whether DDP's per-forward buffer broadcast bumps the model's buffers
(the denoiser's `noise_emb.weight`; a bumped version triggers a re-pack), and what one re-pack costs.

Run under torchrun, one process per GPU:

    torchrun --standalone --nproc_per_node=1 scripts/bench_ddp.py --rounds 3 --steps 10 --warmup 3 --out result.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info(dev):
    import torch

    q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(dev) + " (power limit not readable)"


def cfg2(dev, rank):
    import torch

    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    den = den.to(dev).train()
    den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
    obs, act, _ = frame_stacks(256, 5, 3, 64, 64, 4, 300 + rank)
    batch = types.SimpleNamespace(obs=obs.to(dev), act=act.to(dev), mask_padding=torch.ones(256, 5, dtype=torch.bool, device=dev))
    return den, den.inner_model, lambda m: m(batch)[0], 1.0


def cfg3(dev, rank):
    import torch

    from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig, ActorCriticLossConfig
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, DiffusionSamplerConfig, InnerModelConfig
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    envs, horizon = 32, 15
    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    rem = RewEndModel(RewEndModelConfig(512, 3, 64, 128, [2, 2, 2, 2], [32] * 4, [0] * 4, 4))
    randomize_module_(rem, 2025)
    ac = ActorCritic(ActorCriticConfig(512, 3, 64, [32, 32, 64, 64], [1, 1, 1, 1], 4))
    randomize_module_(ac, 2026)
    den, rem, ac = den.to(dev).eval(), rem.to(dev).eval(), ac.to(dev).train()
    with torch.no_grad():   # P(end) of a few per cent per step, as bench.py's imagination block
        last = [m for m in rem.modules() if isinstance(m, torch.nn.Linear)][-1]
        last.weight[3].fill_(0.05); last.weight[4].fill_(-0.05)
    pool = [frame_stacks(envs, 4, 3, 64, 64, 4, 1000 * (rank + 1) + k)[:2] for k in range(8)]

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
    return ac, ac, lambda m: m()[0], 100.0


WORKLOADS = {"cfg2": cfg2, "cfg3": cfg3}


class SetWeightsCounter:
    """Counts the native `*_set_weights` calls (weight re-packs) made while it is installed."""

    def __init__(self):
        from diamond_b200 import _lib

        self._lib_mod, self.n = _lib, 0
        real, counter = _lib.lib, self

        class Spy:
            def __getattr__(self, k):
                f = getattr(real(), k)
                if not k.endswith("_set_weights"):
                    return f

                def counted(*a):
                    counter.n += 1
                    return f(*a)
                return counted
        self._real, self._spy = real, Spy()

    def __enter__(self):
        self._lib_mod.lib = lambda: self._spy
        return self

    def __exit__(self, *exc):
        self._lib_mod.lib = self._real


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP

    from diamond_b200 import _lib
    from diamond_b200.utils import allreduce_native_gradients

    if "LOCAL_RANK" not in os.environ:
        raise SystemExit("run under torchrun (e.g. torchrun --standalone --nproc_per_node=1 scripts/bench_ddp.py)")
    local, rank, world = int(os.environ["LOCAL_RANK"]), int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    _lib.lib()   # no fallback: raises if the sm_90a library is missing

    def max_over_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    result = {"gpu": gpu_info(dev), "world": world, "rounds": args.rounds, "steps": args.steps, "warmup": args.warmup,
              "direct": "no wrapper; allreduce_native_gradients" + (" issues nothing at world 1" if world == 1 else ""),
              "workloads": {}}
    for name in args.workloads:
        modes = {}
        for mode in ("direct", "ddp"):
            torch.manual_seed(1234 + rank)
            model, native, loss_fn, clip = WORKLOADS[name](dev, rank)
            params = [p for p in model.parameters() if p.requires_grad]
            opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=1e-2, eps=1e-8)
            modes[mode] = dict(model=DDP(model) if mode == "ddp" else model, native=native, loss=loss_fn, clip=clip, params=params,
                               opt=opt, ms=[])

        def step(m):
            m["opt"].zero_grad(set_to_none=True)
            m["loss"](m["model"]).backward()
            if not isinstance(m["model"], DDP):
                allreduce_native_gradients(m["native"])
            torch.nn.utils.clip_grad_norm_(m["params"], m["clip"])
            m["opt"].step()

        for r in range(args.rounds):
            for mode in (("direct", "ddp") if r % 2 == 0 else ("ddp", "direct")):
                m = modes[mode]
                for _ in range(args.warmup):
                    step(m)
                dist.barrier()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    step(m)
                e1.record()
                torch.cuda.synchronize()
                m["ms"].append(max_over_ranks(e0.elapsed_time(e1) / args.steps))
                if rank == 0:
                    print(f"{name} round {r} {mode}: {m['ms'][-1]:.2f} ms/step", flush=True)

        out = {}
        for mode, m in modes.items():
            native = m["native"]
            with SetWeightsCounter() as c:
                step(m)
                torch.cuda.synchronize()
                per_step = c.n
                m["opt"].zero_grad(set_to_none=True)
                m["loss"](m["model"]).backward()          # first micro-step after an optimizer step
                c.n = 0
                versions = [b._version for b in native.buffers()]
                m["loss"](m["model"]).backward()          # second micro-step: weights unchanged since the first
                bumped = sum(b._version != v for b, v in zip(native.buffers(), versions))
                second = c.n
                torch.cuda.synchronize()
            out[mode] = {"ms_per_step": statistics.median(m["ms"]), "ms_per_step_all": m["ms"], "repacks_per_step": per_step,
                         "repacks_in_second_microstep": second, "buffers_bumped_by_a_forward": bumped}
        # one re-pack: the same handle query with and without a parameter version bump in between
        native = modes["direct"]["native"]
        p0 = next(native.parameters())
        native._native()

        def timed(bump, n=20):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                if bump:
                    with torch.no_grad():
                        p0.mul_(1.0)
                native._native()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n
        timed(True, 3)
        repack_ms = max_over_ranks(timed(True) - timed(False))
        out["ddp_over_direct"] = out["ddp"]["ms_per_step"] / out["direct"]["ms_per_step"]
        out["repack_ms"] = repack_ms
        result["workloads"][name] = out
        for m in modes.values():
            m.clear()
        del modes
        torch.cuda.empty_cache()
    if rank == 0:
        print(json.dumps(result))
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(result, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
