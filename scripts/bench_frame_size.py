"""DiffusionSampler.sample() at a frame size beyond 64 x 64: by default the CSGO shape of BASELINE cfg 5 (default net,
150 x 280 RGB, frame stack 4, 10 Euler steps with the default sigmas, 8 images: cfg 5's batch of 64 over 8 GPUs is 8 per GPU,
and imagination has no collective, so one GPU's call is the measurement).  The U-Net runs at 152 x 280 and its mid blocks
attend over 19 x 35 = 665 tokens, the any-L attention path; bench.py measures the 64 x 64 side (8 x 8 = 64 tokens).

The device-resident sample() (CUDA graph) is timed with CUDA events after a warm-up, over at least one second, next to the
reference's GPU path at the same shape and batch (the oracle port of the reference, eager torch with TF32, as bench.py's
gpu_baseline).  Achieved TFLOP/s use FLOP counts computed here from the shapes.  Prints one JSON line; the card, its power
limit and SM clocks are part of it.

    python scripts/bench_frame_size.py [--envs 8] [--hw 150x280] [--warmup 3] [--profile]

--profile adds, from a separate torch.profiler run of one sample(), the kernel time of the attention kernels and their share of
all kernel time in the call."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import torch_oracle as O  # noqa: E402
from diamond_b200.models.diffusion import (Denoiser, DenoiserConfig, DiffusionSampler, DiffusionSamplerConfig,  # noqa: E402
                                           InnerModelConfig)

ATTN_KERNELS = ("attn_qkv_kernel", "attn_stream_kernel", "attn_cluster_kernel")


def flops_per_forward(inner: O.InnerCfg, b: int, h: int, w: int):
    """(conv FLOP, attention FLOP) of one InnerModel forward at b x h x w (2 per multiply-add; real channel counts, the U-Net
    at the padded size as blocks.py:225-229 runs it)."""
    levels = len(inner.depths)
    div = 2 ** (levels - 1)
    hp, wp = -(-h // div) * div, -(-w // div) * div
    ch = inner.channels
    conv = attn = 0.0

    def c3(hw, cin, cout):
        return 2.0 * b * hw * cin * cout * 9

    def block(hw, cin, cout, has_attn):
        nonlocal conv, attn
        conv += c3(hw, cin, cout) + c3(hw, cout, cout) + (2.0 * b * hw * cin * cout if cin != cout else 0.0)
        if has_attn:   # qkv and out projections, q k^T and att v over all heads
            attn += 2.0 * b * hw * (4 * cout * cout) + 4.0 * b * hw * hw * cout

    conv += c3(h * w, (inner.num_steps_conditioning + 1) * inner.img_channels, ch[0])
    for i in range(levels):
        hw = (hp >> i) * (wp >> i)
        if i > 0:
            conv += c3(hw, ch[i - 1], ch[i - 1])
        for k in range(inner.depths[i]):
            block(hw, ch[i - 1 if (k == 0 and i > 0) else i], ch[i], bool(inner.attn_depths[i]))
    hw_mid = (hp >> (levels - 1)) * (wp >> (levels - 1))
    for _ in range(2):
        block(hw_mid, ch[-1], ch[-1], True)
    for i in reversed(range(levels)):
        hw = (hp >> i) * (wp >> i)
        if i < levels - 1:
            conv += c3(hw, ch[i], ch[i])
        c1, c2 = ch[max(0, i - 1)], ch[i]
        n = inner.depths[i]
        for k in range(n + 1):
            block(hw, c2 + (c2 if k < n else c1), c2 if k < n else c1, bool(inner.attn_depths[i]))
    conv += c3(h * w, ch[0], inner.img_channels)
    return conv, attn


def card():
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out["power_limit_sm_clock_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand; the card's limits are then unknown
        out["power_limit_sm_clock_max_sm_clock"] = f"unknown ({e})"
    return out


def timed(fn, warmup, min_s=1.0):
    """ms per call: warm-up, then enough calls for at least min_s seconds, between two CUDA events."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    n = max(3, math.ceil(min_s * 1e3 / max(e0.elapsed_time(e1), 1e-3)))
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8, help="images per sample() (cfg 5: 8 per GPU; 64 for the whole batch on one GPU)")
    ap.add_argument("--hw", default="150x280", help="frame size HxW, e.g. 84x84")
    ap.add_argument("--steps", type=int, default=10, help="Euler denoising steps")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_size: needs a CUDA device")
    h, w = (int(v) for v in a.hw.lower().split("x"))
    b = a.envs
    dev = torch.device("cuda:0")
    inner = O.InnerCfg()
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), 2024)
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels, list(inner.depths),
                                                   list(inner.channels), list(inner.attn_depths), inner.num_actions), 0.5, 0.3))
    den.inner_model.load_state_dict(sd)
    den = den.to(dev).eval()
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(a.steps))
    obs, act, _ = O.synthetic_inputs(b, inner, h, w, 100)
    obs, act = obs.to(dev), act.to(dev)

    conv, attn = flops_per_forward(inner, b, h, w)
    evals = a.steps   # Euler: one denoiser call per step
    levels = len(inner.depths)
    div = 2 ** (levels - 1)
    tokens = (-(-h // div) * div >> (levels - 1)) * (-(-w // div) * div >> (levels - 1))
    out = {"workload": f"sample(), default net, {h}x{w}, {a.steps} Euler steps, {b} images", "envs": b, "attention_tokens": tokens,
           "gflop_conv_per_forward": conv / 1e9, "gflop_attention_per_forward": attn / 1e9}
    with torch.no_grad():
        ms, n = timed(lambda: sampler.sample(obs, act), a.warmup)
    out.update(native_ms_per_sample=ms, timed_calls=n, native_frames_per_s=b / (ms / 1e3),
               native_tflops=(conv + attn) * evals / (ms / 1e3) / 1e12)
    if a.profile:
        from torch.profiler import ProfilerActivity, profile

        with torch.no_grad():
            sampler.sample(obs, act)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                sampler.sample(obs, act)
                torch.cuda.synchronize()
        total = att = 0.0
        for ev in prof.key_averages():
            us = ev.self_device_time_total if hasattr(ev, "self_device_time_total") else ev.self_cuda_time_total
            if ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
                continue
            total += us
            if any(k in ev.key for k in ATTN_KERNELS):
                att += us
        out["profile_kernel_ms"] = total / 1e3
        out["profile_attention_kernel_ms"] = att / 1e3
        out["profile_attention_share"] = att / total if total else None
    # the reference's GPU path: the oracle port of the reference, eager, TF32 (trainer.py:41)
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    cfg = O.DenoiserCfg(inner=inner)
    x0 = torch.randn(b, inner.img_channels, h, w, device=dev)

    def ref_sample():
        with torch.device(dev):   # the oracle creates its per-sample sigma vector on the default device
            O.sample(obs, act, x0, sd_dev, cfg, O.SamplerCfg(a.steps))
    try:
        with torch.no_grad():
            rms, _ = timed(ref_sample, 1)
        out["reference_eager_tf32_ms_per_sample"] = rms
        out["speedup_vs_reference"] = rms / ms
    except torch.cuda.OutOfMemoryError:
        out["reference_eager_tf32_ms_per_sample"] = "out of memory"
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
