"""uint8 vs fp32 frame batches on the GPU: host->device copies, the cfg-2 denoiser step from a host batch, the imagined
environment's pool memory and the two pack kernels.  Each measurement alternates the two paths.  Prints the card and its
power limit first; every number is for that card.

    python scripts/bench_uint8_batches.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from diamond_b200 import frames as F  # noqa: E402
from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig  # noqa: E402
from diamond_b200.synthetic import randomize_module_  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def ms(fn, reps):
    """median ms of fn() (which ends in a device synchronise) over reps calls"""
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def h2d(x, dev):
    def f():
        x.to(dev, non_blocking=x.is_pinned())
        torch.cuda.synchronize()
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    print("card, power limit:", card())
    rng = np.random.default_rng(0)
    shapes = {"cfg-2 denoiser batch 256x5": (256, 5, 3, 64, 64), "rew/end batch 32x19": (32, 19, 3, 64, 64)}
    for name, shp in shapes.items():
        u8 = torch.from_numpy(rng.integers(0, 256, size=shp, dtype=np.uint8))
        f32 = F.cpu_decode(u8)
        res = {}
        for _ in range(2):   # alternate
            for kind, x in (("fp32", f32), ("uint8", u8)):
                for pin in (False, True):
                    y = x.pin_memory() if pin else x
                    h2d(y, dev)()
                    res.setdefault((kind, pin), []).append(ms(h2d(y, dev), a.reps))
        for (kind, pin), v in res.items():
            print(f"h2d {name} {kind:5s} {'pinned' if pin else 'pageable'}: {min(v):.3f} ms ({x.numel() * (4 if kind == 'fp32' else 1) / 1e6:.1f} MB)")

    # the cfg-2 training step end to end from a host batch (pageable, as the trainer copies it)
    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0, 0, 0, 0], 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 1)
    den = den.to(dev).train()
    den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
    u8 = torch.from_numpy(rng.integers(0, 256, size=(256, 5, 3, 64, 64), dtype=np.uint8))
    act = torch.from_numpy(rng.integers(0, 4, size=(256, 5)).astype(np.int64))
    mask = torch.ones(256, 5, dtype=torch.bool)
    host = {"fp32": F.cpu_decode(u8), "uint8": u8}

    def step(obs):
        def f():
            b = SimpleNamespace(obs=obs.to(dev), act=act.to(dev), mask_padding=mask.to(dev))
            den.zero_grad(set_to_none=True)
            loss, _ = den(b)
            loss.backward()
            torch.cuda.synchronize()
        return f
    for k in host:
        for _ in range(3):
            step(host[k])()
    res = {}
    for _ in range(3):
        for k in host:
            res.setdefault(k, []).append(ms(step(host[k]), a.reps))
    for k, v in res.items():
        print(f"cfg-2 step from a host batch, {k:5s}: {min(v):.2f} ms (best of 3 medians over {a.reps})")

    # pool memory: 256 preloaded batches x 32 envs x 4 frames, as WorldModelEnv keeps them
    for k in ("fp32", "uint8"):
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        pool = [torch.empty(32, 4, 3, 64, 64, dtype=torch.float32 if k == "fp32" else torch.uint8, device=dev) for _ in range(256)]
        pool = torch.cat(pool)
        if k == "uint8":
            kinds = torch.ones(pool.shape[:2], dtype=torch.uint8, device=dev)
        print(f"pool {k:5s}: {(torch.cuda.max_memory_allocated() - base) / 1e9:.3f} GB peak while filling, {pool.numel() * pool.element_size() / 1e9:.3f} GB held")
        del pool

    # the two pack kernels, by torch.profiler on the denoiser no-grad forward and the rew/end prediction
    from torch.profiler import ProfilerActivity, profile
    im = den.inner_model
    b = 256
    lv = u8.to(dev)
    kinds = torch.ones(b, 5, dtype=torch.uint8, device=dev)
    noisy = torch.randn(b, 3, 64, 64, device=dev)
    cn = torch.randn(b, device=dev)
    obs_f = (F.decode(lv[:, :4], kinds[:, :4]) / 0.5).reshape(b, 12, 64, 64)
    stack = F.U8FrameStack(lv[:, :4], kinds[:, :4], F.context_table(dev, 0.5))
    with torch.no_grad():
        for _ in range(3):
            im(noisy, cn, obs_f, act[:, :4].to(dev)); im(noisy, cn, stack, act[:, :4].to(dev))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                im(noisy, cn, obs_f, act[:, :4].to(dev)); im(noisy, cn, stack, act[:, :4].to(dev))
            torch.cuda.synchronize()
    for e in prof.key_averages():
        if "pack_denoiser_input" in e.key or "pack_rew_end" in e.key:
            print(f"kernel {e.key[:90]}: {getattr(e, "device_time_total", 0) / max(e.count, 1):.1f} us x {e.count}")


if __name__ == "__main__":
    main()
