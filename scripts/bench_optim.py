"""clip_grad_norm_ + AdamW over each trained model's parameters: torch's default (foreach, the optimizer `utils.configure_opt`
builds), torch `fused=True`, and the native kernels (diamond_b200.optim), in alternation on the same gradients.

Per model (default config, gradients from one native backward at the trainer's shapes, max_norm as trainer.yaml):
  - device_us: CUDA events around clip + step with the host's launches queued behind a spin kernel, i.e. GPU time alone;
  - step_us: CUDA events around clip + step from an idle GPU, i.e. including the host's time to issue the launches;
  - kernel_us and launches per step: the CUDA kernels of 20 steps under torch.profiler (native: also dmd_launch_count);
  - bytes the native kernels move (40 B per parameter with the clip active: the norm reads g, the scale reads and writes it,
    AdamW reads p, g, m, v and writes p, m, v; 32 B when the coefficient is 1 and the scale touches nothing) and the rate
    over kernel_us against the 3.35 TB/s of the H100 SXM data sheet.
The gradients are restored before every step, outside the timed window, so every arm clips the same gradients.
Then the cfg-2 denoiser training step (B = 256) and the 32 x 19 reward/termination step end to end with each optimizer.
Prints one JSON line; the card, its power limit and SM clock are read in the same run.

    python scripts/bench_optim.py [--steps 200] [--warmup 20] [--e2e-steps 10]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from diamond_b200 import _lib, optim  # noqa: E402
from oracle import optim_reference as OR  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
ARMS = ("torch_foreach", "torch_fused", "native")


class _Batch:
    pass


def models(dev):
    """name -> (module, max_norm, one_backward): each model at its default config, gradients at the trainer's shapes."""
    from bench_rew_end_train import _Batch as RBatch, inputs as rew_end_inputs
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    den = den.to(dev).train()
    den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
    obs, act, _ = frame_stacks(256, 5, 3, 64, 64, 4, 300)
    b = _Batch()
    b.obs, b.act, b.mask_padding = obs.to(dev), act.to(dev), torch.ones(256, 5, dtype=torch.bool, device=dev)

    def den_backward():
        den(b)[0].backward()

    rem = RewEndModel(RewEndModelConfig(512, 3, 64, 128, [2, 2, 2, 2], [32] * 4, [0] * 4, 4))
    randomize_module_(rem, 2025)
    rem = rem.to(dev).train()
    r_obs, r_act, r_rew, r_end, r_mask, final_obs = rew_end_inputs(32, 19, dev)
    info = [{"final_observation": final_obs[i]} if i in final_obs else {} for i in range(32)]

    def rem_backward():
        rem(RBatch(r_obs.clone(), r_act, r_rew, r_end, r_mask, info))[0].backward()

    ac = ActorCritic(ActorCriticConfig(512, 3, 64, [32, 32, 64, 64], [1, 1, 1, 1], 4))
    randomize_module_(ac, 2026)
    ac = ac.to(dev).train()
    gen = torch.Generator(device=dev).manual_seed(5)
    frames = torch.rand(15, 32, 3, 64, 64, generator=gen, device=dev) * 2 - 1

    def ac_backward():   # 32 envs x horizon 15 through the native policy, BPTT through its LSTM
        hx = cx = torch.zeros(32, 512, device=dev)
        loss = 0.0
        for t in range(15):
            out = ac.predict_act_value(frames[t], (hx, cx))
            hx, cx = out.hx_cx
            loss = loss + out.logits_act.logsumexp(-1).mean() + out.val.pow(2).mean()
        loss.backward()

    return {"denoiser": (den, 1.0, den_backward), "rew_end": (rem, 100.0, rem_backward), "actor_critic": (ac, 100.0, ac_backward)}


def make_opt(arm, model):
    groups = OR.configure_opt_groups(model, 1e-2)
    if arm == "native":
        return optim.AdamW(groups, lr=1e-4, eps=1e-8)
    return torch.optim.AdamW(groups, lr=1e-4, eps=1e-8, **({"fused": True} if arm == "torch_fused" else {}))


def clip_fn(arm):
    return optim.clip_grad_norm_ if arm == "native" else torch.nn.utils.clip_grad_norm_


def kernel_profile(step, restore, n=20):
    """(CUDA kernels per step, their summed time per step in us) over n steps under torch.profiler, the gradient restore
    included (step=None profiles the restore alone, to subtract)."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            restore()
            torch.cuda.synchronize()
            if step is not None:
                step()
        torch.cuda.synchronize()
    count = us = 0
    for ev in prof.key_averages():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.key.startswith(("Memcpy", "Memset")):
            continue
        count += ev.count
        us += ev.self_device_time_total
    return count / n, us / n


def bench_optimizer(name, model, max_norm, backward, steps, warmup):
    params = [p for p in model.parameters() if p.requires_grad]
    model.zero_grad(set_to_none=True)
    backward()
    grads = [p.grad for p in params]
    saved = [g.clone() for g in grads]
    n = sum(p.numel() for p in params)
    opts = {arm: make_opt(arm, model) for arm in ARMS}
    steps_fn = {arm: (lambda arm=arm: (clip_fn(arm)(params, max_norm), opts[arm].step())) for arm in ARMS}
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    dev_us = {a: 0.0 for a in ARMS}
    step_us = {a: 0.0 for a in ARMS}
    for it in range(warmup + steps):
        for arm in ARMS:
            for mode in ("device", "step"):
                torch._foreach_copy_(grads, saved)
                torch.cuda.synchronize()
                e0, e1 = ev(), ev()
                if mode == "device":
                    torch.cuda._sleep(10_000_000)   # ~5 ms of spin: the launches below queue up behind it
                e0.record()
                steps_fn[arm]()
                e1.record()
                torch.cuda.synchronize()
                if it >= warmup:
                    (dev_us if mode == "device" else step_us)[arm] += e0.elapsed_time(e1) * 1e3 / steps
    torch._foreach_copy_(grads, saved)
    norm = float(torch.nn.utils.get_total_norm(saved))
    lib = _lib.lib()
    lib.dmd_launch_count(1)
    steps_fn["native"]()
    dmd_launches = lib.dmd_launch_count(1)
    restore = lambda: torch._foreach_copy_(grads, saved)  # noqa: E731
    base_n, base_us = kernel_profile(None, restore)
    launches, kernel_us = {}, {}
    for arm in ARMS:
        k, us = kernel_profile(steps_fn[arm], restore)
        launches[arm], kernel_us[arm] = round(k - base_n, 2), us - base_us
    nbytes = (40 if norm > max_norm else 32) * n
    out = {"params": n, "tensors": len(params), "max_norm": max_norm, "grad_norm": norm, "clip_active": norm > max_norm,
           "device_us": dev_us, "step_us": step_us, "kernel_us": kernel_us, "launches_per_step": launches,
           "native_dmd_launch_count": dmd_launches, "native_bytes": nbytes,
           "native_GBps_over_kernel_us": nbytes / (kernel_us["native"] * 1e-6) / 1e9,
           "native_fraction_of_3.35TBps": nbytes / (kernel_us["native"] * 1e-6) / HBM_BYTES_PER_S,
           "bound_us_at_3.35TBps": nbytes / HBM_BYTES_PER_S * 1e6}
    print(f"{name}: {json.dumps(out)}", file=sys.stderr)
    return out


def bench_training_step(name, model, max_norm, backward, steps, warmup):
    """zero_grad + forward + backward + clip + step, each optimizer in turn, CUDA events around the whole step."""
    params = [p for p in model.parameters() if p.requires_grad]
    opts = {arm: make_opt(arm, model) for arm in ARMS}
    ms = {a: 0.0 for a in ARMS}
    for it in range(warmup + steps):
        for arm in ARMS:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            opts[arm].zero_grad(set_to_none=True)
            backward()
            clip_fn(arm)(params, max_norm)
            opts[arm].step()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                ms[arm] += e0.elapsed_time(e1) / steps
    print(f"{name} training step ms: {json.dumps(ms)}", file=sys.stderr)
    return ms


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand; the card's settings are then unknown
        q = f"unknown ({e})"
    return {"gpu": torch.cuda.get_device_name(0), "name_power_limit_sm_clock_max_sm_clock": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--e2e-steps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim: needs a CUDA device")
    dev = torch.device("cuda:0")
    ms = models(dev)
    out = {"workload": "clip_grad_norm_ + AdamW per model: torch foreach / torch fused / native", "card_before": card()}
    for name, (model, max_norm, backward) in ms.items():
        out[name] = bench_optimizer(name, model, max_norm, backward, a.steps, a.warmup)
    for name in ("denoiser", "rew_end"):
        model, max_norm, backward = ms[name]
        out[name]["training_step_ms"] = bench_training_step(name, model, max_norm, backward, a.e2e_steps, 2)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
