"""One reward / termination training step at the trainer's shape (trainer.yaml:108,113: 32 segments x seq_length 19, i.e.
18 transitions and 576 encoder rows per segment batch): RewEndModel.forward + backward + clip_grad_norm_(100) + AdamW, timed
with CUDA events after a warm-up, next to the same step on the reference's GPU path (the oracle port of the reference model,
eager torch with TF32, as bench.py's gpu_baseline).  Prints one JSON line; the card and its power limit are part of it.

    python scripts/bench_rew_end_train.py [--steps 20] [--warmup 5] [--profile]

--profile adds the native step's kernel time per part (torch.profiler, CUDA activity, kernels classified by name: the LSTM /
head kernels are the fp32 GEMM, linear, LSTM-cell, SiLU-adjoint and logits kernels; everything else is the encoder)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import torch_oracle as O  # noqa: E402
from oracle import rew_end_training as RT  # noqa: E402
from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig  # noqa: E402

LSTM_HEAD_KERNELS = ("sgemm_kernel", "splitk_reduce", "linear_kernel", "lstm_", "dsilu_mul", "merge_logits", "split_logits",
                     "nhwc_to_nchw_kernel", "colsum_kernel")


class _Batch:
    def __init__(self, obs, act, rew, end, mask, info):
        self.obs, self.act, self.rew, self.end, self.mask_padding, self.info = obs, act, rew, end, mask, info
        self.trunc = torch.zeros_like(end)


def inputs(b, T, dev):
    cfg = O.RewEndCfg()
    rng = np.random.default_rng(1901)
    obs = RT.frames(rng.integers(0, 256, size=(b, T, cfg.img_channels, cfg.img_size, cfg.img_size), dtype=np.uint8)).to(dev)
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, T))).to(dev)
    rew = torch.from_numpy(rng.choice([-1.0, 0.0, 0.0, 1.0], size=(b, T)).astype(np.float32)).to(dev)
    end = torch.zeros(b, T, dtype=torch.long, device=dev)
    mask = torch.ones(b, T, dtype=torch.bool, device=dev)
    end[1, 9] = 1
    mask[1, 10:] = False
    final_obs = {1: obs[1, 10].clone()}
    return obs, act, rew, end, mask, final_obs


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--segments", type=int, default=32)
    ap.add_argument("--seq-length", type=int, default=19)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rew_end_train: needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 779)
    model = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                          list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
    model.load_state_dict(sd)
    model = model.to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    obs, act, rew, end, mask, final_obs = inputs(a.segments, a.seq_length, dev)
    info = [{"final_observation": final_obs[i]} if i in final_obs else {} for i in range(a.segments)]

    def batch():
        return _Batch(obs.clone(), act, rew, end, mask, info)

    def native_step():
        opt.zero_grad(set_to_none=True)
        loss, _ = model(batch())
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 100.0)
        opt.step()

    def native_fwd_bwd():
        loss, _ = model(batch())
        loss.backward()

    def optimizer():
        torch.nn.utils.clip_grad_norm_(model.parameters(), 100.0)
        opt.step()

    out = {"workload": f"rew_end training step, {a.segments} x {a.seq_length}", "rows": a.segments * (a.seq_length - 1)}
    out["native_ms_per_step"] = timed(native_step, a.steps, a.warmup)
    out["native_segments_per_s"] = a.segments / (out["native_ms_per_step"] / 1e3)
    out["native_forward_backward_ms"] = timed(native_fwd_bwd, a.steps, a.warmup)
    out["optimizer_ms"] = timed(optimizer, a.steps, a.warmup)
    if a.profile:
        from torch.profiler import ProfilerActivity, profile

        native_step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            native_fwd_bwd()
            torch.cuda.synchronize()
        enc = lstm = 0.0
        for ev in prof.key_averages():
            us = ev.self_device_time_total if hasattr(ev, "self_device_time_total") else ev.self_cuda_time_total
            if any(k in ev.key for k in LSTM_HEAD_KERNELS):
                lstm += us
            elif ev.key.startswith("Memcpy") or ev.key.startswith("Memset") or "cross_entropy" in ev.key or "elementwise" in ev.key:
                continue
            else:
                enc += us
        out["kernel_ms_encoder"] = enc / 1e3
        out["kernel_ms_lstm_and_head"] = lstm / 1e3
    # the reference's GPU path: the oracle port of the reference model, eager, TF32 (trainer.py:41)
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    sd_ref = {k: v.to(dev).requires_grad_(True) for k, v in O.seeded_state_dict(O.rew_end_shapes(cfg), 779).items()}
    opt_ref = torch.optim.AdamW(list(sd_ref.values()), lr=1e-4, weight_decay=1e-2, eps=1e-8)

    def ref_step():
        opt_ref.zero_grad(set_to_none=True)
        with torch.device(dev):   # the oracle creates its zero LSTM state on the default device
            loss = RT.rew_end_loss(obs, act, rew, end, mask, final_obs, sd_ref, cfg)[0]
        loss.backward()
        torch.nn.utils.clip_grad_norm_(list(sd_ref.values()), 100.0)
        opt_ref.step()
    try:
        out["reference_eager_tf32_ms_per_step"] = timed(ref_step, max(3, a.steps // 4), 2)
        out["speedup_vs_reference"] = out["reference_eager_tf32_ms_per_step"] / out["native_ms_per_step"]
    except torch.cuda.OutOfMemoryError:
        out["reference_eager_tf32_ms_per_step"] = "out of memory"
    out["gpu"] = torch.cuda.get_device_name(0)
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers stand; the card's limit is then unknown
        out["power_limit"] = f"unknown ({e})"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
