"""DiffusionSampler.sample() with 128-channel U-Net levels next to the default net: [64, 64, 64, 64] (the default),
[64, 128, 128, 128] and [128] * 4, each with the default depths, 64 x 64 RGB frames, frame stack 4, 32 images and 3 Euler steps
(the default sampler), and a cfg-2 training step (Denoiser.forward + backward + clip + AdamW, frame stack 4 + 1 autoregressive
step, batch 256 as bench.py).  The 128 -> 128 convs and the 256-channel up-path concats run K-split, the mid-block attention at
C = 128.

Each net's device-resident sample() (CUDA graph) and training step are timed with CUDA events after a warm-up.
Achieved TFLOP/s use FLOP counts computed from the shapes (scripts/bench_frame_size.py).  Prints one JSON line per net; the
card, its power limit and SM clocks are part of each.

    python scripts/bench_wide_levels.py [--envs 32] [--steps 3] [--warmup 3] [--train-batch 256]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_frame_size import card, flops_per_forward, timed  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402
from diamond_b200.models.diffusion import (Denoiser, DenoiserConfig, DiffusionSampler, DiffusionSamplerConfig,  # noqa: E402
                                           InnerModelConfig, SigmaDistributionConfig)
from diamond_b200.synthetic import frame_stacks  # noqa: E402

NETS = {"default": [64, 64, 64, 64], "wide": [64, 128, 128, 128], "wide128": [128, 128, 128, 128]}


def train_step_ms(den, batch, dev, steps=5, warmup=2):
    """ms per Denoiser.forward + backward + clip_grad_norm_ + AdamW step (bench.py train_block, one GPU)."""
    den.train()
    den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
    opt = torch.optim.AdamW(den.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    obs, act, _ = frame_stacks(batch, 5, 3, 64, 64, 4, 300)

    class B_:
        pass

    b = B_()
    b.obs, b.act, b.mask_padding = obs.to(dev), act.to(dev), torch.ones(batch, 5, dtype=torch.bool, device=dev)

    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = den(b)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(den.parameters(), 1.0)
        opt.step()
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    den.eval()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=32)
    ap.add_argument("--steps", type=int, default=3, help="Euler denoising steps")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--train-batch", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wide_levels: needs a CUDA device")
    dev = torch.device("cuda:0")
    b, h, w = a.envs, 64, 64
    info = card()
    for name, channels in NETS.items():
        inner = O.InnerCfg(channels=channels)
        sd = O.seeded_state_dict(O.inner_model_shapes(inner), 2025)
        den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                       list(inner.depths), list(inner.channels), list(inner.attn_depths), inner.num_actions),
                                      0.5, 0.3))
        den.inner_model.load_state_dict(sd)
        den = den.to(dev).eval()
        sampler = DiffusionSampler(den, DiffusionSamplerConfig(a.steps))
        obs, act, _ = O.synthetic_inputs(b, inner, h, w, 100)
        obs, act = obs.to(dev), act.to(dev)
        conv, attn = flops_per_forward(inner, b, h, w)
        with torch.no_grad():
            ms, n = timed(lambda: sampler.sample(obs, act), a.warmup)
        out = {"workload": f"sample(), channels {channels}, {h}x{w}, {a.steps} Euler steps, {b} images", "net": name,
               "gflop_per_forward": (conv + attn) / 1e9, "ms_per_sample": ms, "timed_calls": n, "frames_per_s": b / (ms / 1e3),
               "tflops": (conv + attn) * a.steps / (ms / 1e3) / 1e12}
        out["train_ms_per_step"] = train_step_ms(den, a.train_batch, dev)
        out["train_batch"] = a.train_batch
        out.update(info)
        print(json.dumps(out), flush=True)
        del den, sampler
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
