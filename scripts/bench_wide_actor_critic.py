"""Actor-critics with 128-channel levels on the GPU: per policy config, at `--envs` x `--horizon`,
  - forward time per imagined step (one dmd_actor_critic_forward at B = envs, as each autograd node of the rollout runs it);
  - backward time per rollout (loss.backward() through `horizon` BPTT nodes);
  - the whole cfg-3 update (ActorCritic.forward() over WorldModelEnv: native sampler with 3 denoising steps, native
    reward / termination model, native policy; then backward, clip and AdamW), as bench.py's imagination block runs it, in
    rounds that alternate the policies (median, min and max over the rounds).  The reference's GPU path is measured for the
    policy's own update only, not for the whole update;
  - the policy's own update over pre-generated frames (rollout + loss + backward), native and on the reference's GPU path
    (the oracle port run eagerly on cuda, fp32 with TF32 matmul as src/trainer.py:41);
  - the per-node workspace and backward-scratch bytes, and the peak device memory the whole update allocates over what the
    process already holds (the world model, every policy and its environment).
The GPU's name, power limit and SM clocks are read before and after.  Prints one JSON object.

--trace runs torch.profiler (CUDA kernels) instead: one forward and one backward node of --trace-config at B = envs, with
the share of kernel time in its K-split conv passes and dgrad chunks, and one 3x3 128 -> 128 conv at each level's frame size
in both K-split policies (three passes per 64-channel chunk, or one launch per 16-channel chunk).

--dump-outputs DIR writes the default [32, 32, 64, 64] policy's forward outputs and one backward's flat gradient at fixed
seeds (B = 32, through the C ABI only) as .npy files, with the kernel launches per forward and per backward, and exits.  With
--lib it runs against another build of the library, so two builds' dumps can be compared byte for byte.

    python scripts/bench_wide_actor_critic.py [--configs 64,128,128,128 128,128,128,128] [--envs 32 --horizon 15]
    python scripts/bench_wide_actor_critic.py --trace [--trace-config 128,128,128,128]
    python scripts/bench_wide_actor_critic.py --dump-outputs /tmp/ac_dump [--lib path/to/libdiamond_b200.so]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:  # the measurement stands without it, but says so
        return {"error": repr(e)}


def ac_config(channels, envs_img=64):
    from diamond_b200.models.actor_critic import ActorCriticConfig

    return ActorCriticConfig(512, 3, envs_img, list(channels), [1] * len(channels), 4)


def seeded_ac(channels, seed, dev):
    from diamond_b200.models.actor_critic import ActorCritic
    from oracle import torch_oracle as O

    cfg = O.ActorCriticCfg(channels=list(channels))
    ac = ActorCritic(ac_config(channels))
    ac.load_state_dict(O.seeded_actor_critic_state_dict(cfg, seed))
    return ac.to(dev).train(), cfg


def abi_node(ac, b, seed, dev):
    """One autograd node through the C ABI at B = b with seeded inputs: (forward(), backward(), [logits, val, hx, cx],
    [g_hx_in, g_cx_in], flat gradient)."""
    import torch

    from diamond_b200 import _lib

    lib = _lib.lib()
    h = ac._native()
    gen = torch.Generator().manual_seed(seed)
    obs = (torch.rand(b, 3, 64, 64, generator=gen) * 2 - 1).to(dev)
    hx, cx = (torch.randn(b, 512, generator=gen) * 0.3).to(dev), (torch.randn(b, 512, generator=gen) * 0.3).to(dev)
    g_out = [torch.randn(b, 4, generator=gen).to(dev), torch.randn(b, generator=gen).to(dev),
             torch.randn(b, 512, generator=gen).to(dev), torch.randn(b, 512, generator=gen).to(dev)]
    ws = torch.zeros(lib.dmd_actor_critic_workspace_bytes(h, b), dtype=torch.uint8, device=dev)
    scratch = torch.zeros(lib.dmd_actor_critic_backward_scratch_bytes(h, b), dtype=torch.uint8, device=dev)
    out = [torch.zeros(b, 4, device=dev), torch.zeros(b, device=dev), torch.zeros_like(hx), torch.zeros_like(cx)]
    g_in = [torch.zeros_like(hx), torch.zeros_like(cx)]
    flat = torch.zeros(ac._grad_views_layout()[2], device=dev)
    st = _lib.current_stream()

    def forward():
        _lib.check(lib.dmd_actor_critic_forward(h, b, obs.data_ptr(), hx.data_ptr(), cx.data_ptr(), *[o.data_ptr() for o in out],
                                                ws.data_ptr(), ws.numel(), st))

    def backward():
        _lib.check(lib.dmd_actor_critic_backward(h, b, hx.data_ptr(), cx.data_ptr(), out[2].data_ptr(), *[g.data_ptr() for g in g_out],
                                                 flat.data_ptr(), flat.numel(), g_in[0].data_ptr(), g_in[1].data_ptr(), ws.data_ptr(),
                                                 scratch.data_ptr(), scratch.numel(), st))
    return forward, backward, out, g_in, flat


def dump_outputs(out_dir, dev):
    import numpy as np
    import torch

    from diamond_b200 import _lib

    os.makedirs(out_dir, exist_ok=True)
    lib = _lib.lib()
    ac, _ = seeded_ac([32, 32, 64, 64], 2026, dev)
    forward, backward, out, g_in, flat = abi_node(ac, 32, 2027, dev)
    forward()   # weights packed on the first call
    torch.cuda.synchronize()
    lib.dmd_launch_count(1)
    forward()
    n_fwd = lib.dmd_launch_count(1)
    backward()
    n_bwd = lib.dmd_launch_count(1)
    torch.cuda.synchronize()
    digests = {}
    for name, t in zip(["logits", "val", "hx", "cx", "g_hx_in", "g_cx_in", "grad"], out + g_in + [flat]):
        a = t.cpu().numpy()
        np.save(os.path.join(out_dir, name + ".npy"), a)
        digests[name] = hashlib.sha256(a.tobytes()).hexdigest()[:16]
    res = {"lib": _lib.LIB_PATH, "launches_per_forward": n_fwd, "launches_per_backward": n_bwd, "sha256": digests}
    with open(os.path.join(out_dir, "launches.json"), "w") as f:
        json.dump(res, f)
    return res


def timed(fn, n):
    import torch

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def scripted_frames(envs, horizon, dev, seed):
    import torch

    gen = torch.Generator().manual_seed(seed)
    return (torch.randint(0, 256, (horizon + 1, envs, 3, 64, 64), generator=gen).float() / 255 * 2 - 1).to(dev)


class ScriptedEnv:
    """Pre-generated frames, no episode ends: the policy's own share of an imagination update."""

    def __init__(self, frames):
        self.frames, self.t = frames, 0
        self.num_envs, self.num_actions = frames.size(1), 4
        z = self.frames.new_zeros(self.num_envs)
        self.rew, self.flag = z, z.long()

    def reset(self, seed=None):
        self.t = 0
        return self.frames[0], {}

    def step(self, act):
        self.t += 1
        return self.frames[self.t % self.frames.size(0)], self.rew, self.flag, self.flag, {}


def policy_update_ms(ac, frames, horizon, reps):
    import torch

    from diamond_b200.models.actor_critic import ActorCriticLossConfig

    ac.env_loop = ac.loss_cfg = None
    ac.setup_training(ScriptedEnv(frames), ActorCriticLossConfig(horizon, 0.985, 0.95, 1.0, 0.001))

    def step():
        loss, _ = ac()
        loss.backward()
        ac.zero_grad(set_to_none=True)
    step()
    return timed(step, reps)


def reference_policy_update_ms(cfg, frames, horizon, reps, dev):
    """The oracle port of ActorCritic.forward + backward on cuda, eager, fp32 with TF32 matmul."""
    import torch

    from oracle import torch_oracle as O

    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    sd = {k: v.to(dev).requires_grad_(True) for k, v in O.seeded_actor_critic_state_dict(cfg, 2026).items()}
    b = frames.size(1)
    flags = torch.zeros(horizon, b, dtype=torch.long)
    act = torch.zeros(b, horizon, dtype=torch.long, device=dev)
    rew = torch.zeros(b, horizon, device=dev)
    lc = O.ActorCriticLossCfg(backup_every=horizon)

    def step():
        hx = torch.zeros(b, cfg.lstm_dim, device=dev)
        logits, val, vb = O.actor_critic_rollout(frames, flags, flags, {}, sd, cfg, hx, hx.clone())
        f = flags.t().to(dev).float()
        loss, _ = O.actor_critic_loss(logits, val, act, rew, f, f, vb, lc)
        loss.backward()
        for v in sd.values():
            v.grad = None
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
    try:
        step()
        return timed(step, reps)
    finally:   # the later measurements of this process run with the flags as they were
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def backward_per_rollout_ms(ac, frames, horizon, reps):
    import torch

    def rollout():
        b = frames.size(1)
        hx = torch.zeros(b, 512, device=frames.device)
        cx = torch.zeros_like(hx)
        loss = 0
        for t in range(horizon):
            logits, val, (hx, cx) = ac.predict_act_value(frames[t], (hx, cx))
            loss = loss + logits.sum() + val.sum()
        return loss
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    total = 0.0
    for i in range(reps + 1):
        loss = rollout()
        torch.cuda.synchronize()
        e0, e1 = ev(), ev()
        e0.record()
        loss.backward()
        e1.record()
        torch.cuda.synchronize()
        ac.zero_grad(set_to_none=True)
        if i:
            total += e0.elapsed_time(e1)
    return total / reps


def world_model(envs, dev):
    """The denoiser, reward / termination model and in-memory loader of bench.py's imagination block (cfg 3)."""
    import torch

    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    rem = RewEndModel(RewEndModelConfig(512, 3, 64, 128, [2, 2, 2, 2], [32] * 4, [0] * 4, 4))
    randomize_module_(rem, 2025)
    den, rem = den.to(dev).eval(), rem.to(dev).eval()
    with torch.no_grad():   # rare episode ends, as bench.py
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
    return den, rem, Loader()


class WholeUpdate:
    """bench.py's imagination block (cfg 3) with a given policy, on its own WorldModelEnv over the shared world model."""

    def __init__(self, ac, wm, horizon):
        import torch

        from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
        from diamond_b200.models.actor_critic import ActorCriticLossConfig
        from diamond_b200.models.diffusion import DiffusionSamplerConfig

        self.ac = ac
        ac.env_loop = ac.loss_cfg = None
        ac.setup_training(WorldModelEnv(*wm, WorldModelEnvConfig(horizon, 4, DiffusionSamplerConfig(3))),
                          ActorCriticLossConfig(horizon, 0.985, 0.95, 1.0, 0.001))
        self.opt = torch.optim.AdamW(ac.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)

    def step(self):
        import torch

        self.opt.zero_grad(set_to_none=True)
        loss, _ = self.ac()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(self.ac.parameters(), 100.0)
        self.opt.step()

    def block(self, updates, dev):
        """One warm-up update, then `updates` timed ones: (ms per update, peak device bytes above what was allocated when the
        block started).  The policy's workspace pool and backward scratch are released first, so the peak counts what its
        updates allocate (rollout workspaces, scratch, gradients) over the models and environments every policy keeps."""
        import torch

        self.ac.__dict__.pop("_ws_pool", None)
        self.ac.__dict__.pop("_bwd_scratch", None)
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        self.step()
        ms = timed(self.step, updates)
        return ms, int(torch.cuda.max_memory_allocated(dev) - base)


def bench_config(channels, args, dev):
    from diamond_b200 import _lib

    lib = _lib.lib()
    ac, cfg = seeded_ac(channels, 2026, dev)
    h = ac._native()
    frames = scripted_frames(args.envs, args.horizon, dev, 7)
    import torch

    ws = torch.empty(lib.dmd_actor_critic_workspace_bytes(h, args.envs), dtype=torch.uint8, device=dev)
    hx = torch.zeros(args.envs, 512, device=dev)
    timed(lambda: ac._native_forward(frames[0], hx, hx, ws), 5)   # warm-up (and the weight packing of the first call)
    fwd_ms = timed(lambda: ac._native_forward(frames[0], hx, hx, ws), 200)
    out = {"channels": list(channels),
           "workspace_bytes_per_node": int(lib.dmd_actor_critic_workspace_bytes(h, args.envs)),
           "backward_scratch_bytes": int(lib.dmd_actor_critic_backward_scratch_bytes(h, args.envs)),
           "forward_ms_per_imagined_step": fwd_ms,
           "backward_ms_per_rollout": backward_per_rollout_ms(ac, frames, args.horizon, args.reps),
           "policy_update_ms_native": policy_update_ms(ac, frames, args.horizon, args.reps),
           "policy_update_ms_reference_gpu_path": reference_policy_update_ms(cfg, frames, args.horizon, args.reps, dev)}
    ac.__dict__.pop("_ws_pool", None)
    del ws
    torch.cuda.empty_cache()
    return ac, out


def whole_updates(acs, results, args, dev):
    """The whole cfg-3 update of every policy, in `--whole-repeats` rounds that alternate the policies (the world model's
    share dominates it, and its run-to-run spread is larger than a policy's share).  There is no reference-path number for
    the whole update: the reference's GPU path is measured for the policy's own update only."""
    wm = world_model(args.envs, dev)
    runs = [WholeUpdate(ac, wm, args.horizon) for ac in acs]
    times = [[] for _ in acs]
    peaks = [0 for _ in acs]
    for _ in range(args.whole_repeats):
        for i, r in enumerate(runs):
            ms, peak = r.block(args.updates, dev)
            times[i].append(ms)
            peaks[i] = max(peaks[i], peak)
    for res, t, p in zip(results, times, peaks):
        res.update(whole_update_ms_per_round=t, whole_update_ms_median=sorted(t)[len(t) // 2], whole_update_ms_min=min(t),
                   whole_update_ms_max=max(t), whole_update_peak_bytes_above_start=p, whole_update_reference_gpu_path="not measured")


# ------------------------------------------------------------------------------------------------ kernel traces
def _cuda_kernels(prof):
    """(name, start us, duration us) of every CUDA kernel in a torch.profiler run, in launch order."""
    from torch.autograd import DeviceType

    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    return [(e.name, e.time_range.start, e.time_range.elapsed_us()) for e in ev]


def _profile(fn, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return _cuda_kernels(prof)


def _by_class(kernels):
    out = {}
    for name, _, us in kernels:
        k = "conv_tc_kernel" if "conv_tc_kernel" in name else "wgrad" if "wgrad" in name else name.split("(")[0].split("<")[0].replace("void ", "")
        out[k] = out.get(k, 0.0) + us
    return out


def trace_policy(channels, b, reps, dev):
    """torch.profiler trace of one forward and one backward node at B = b through the C ABI: kernel time per class, and the
    share of the conv launches.  In a policy whose levels are all 128 -> 128 ([128] * 4), every forward conv launch after
    conv0 is a pass of a K-split conv, and every backward conv launch is a dgrad chunk."""
    ac, _ = seeded_ac(channels, 2026, dev)
    forward, backward, *_ = abi_node(ac, b, 2028, dev)
    res = {}
    for name, fn in (("forward", forward), ("backward", lambda: (forward(), backward()))):
        k = _profile(fn, reps)
        if name == "backward":   # keep the backward's kernels only: drop each repetition's forward
            fk = _profile(forward, reps)
            per_fwd = len(fk) // reps
            per = len(k) // reps
            k = [x for i, x in enumerate(k) if i % per >= per_fwd]
        total = sum(us for _, _, us in k) / reps
        convs = [us for n, _, us in k if "conv_tc_kernel" in n]
        per_rep = len(convs) // reps
        if name == "forward":   # conv0 is each repetition's first conv launch
            ksplit = [us for i, us in enumerate(convs) if i % per_rep != 0]
        else:
            ksplit = convs
        res[name] = {"kernel_us": total, "kernels_per_call": len(k) // reps,
                     "conv_launches_per_call": per_rep, "k_split_or_dgrad_chunk_launches_per_call": len(ksplit) // reps,
                     "k_split_or_dgrad_chunk_us": sum(ksplit) / reps, "share": sum(ksplit) / reps / total,
                     "by_class_us": {c: v / reps for c, v in sorted(_by_class(k).items(), key=lambda kv: -kv[1])}}
    return res


def trace_chunk_policies(b, sizes, reps, dev):
    """One 3x3 128 -> 128 split-fp16 conv at B = b and each frame size, traced in both K-split policies on the same operand:
    three passes per 64-channel chunk (6 launches, the library's plan) and one K = 3 x 16 launch per 16-channel chunk
    (8 launches, the alternative of 8 one-launch chunks).  Both are checked against a float32 cuDNN conv first."""
    import ctypes as C

    import torch
    import torch.nn.functional as F

    from diamond_b200 import _lib

    lib = _lib.lib()
    st = _lib.current_stream()
    gen = torch.Generator().manual_seed(2029)
    w = (torch.randn(128, 128, 3, 3, generator=gen) * 0.03).to(dev)
    bias = (torch.randn(128, generator=gen) * 0.1).to(dev)
    half = lambda n: torch.empty(n, dtype=torch.float16, device=dev)  # noqa: E731
    pk_hi, pk_lo, pk_16 = [half(9 * 64 * 128) for _ in range(2)], [half(9 * 64 * 128) for _ in range(2)], [half(3 * 9 * 16 * 128) for _ in range(8)]
    for j in range(2):
        _lib.check(lib.dmd_pack_conv_weight(w.data_ptr(), pk_hi[j].data_ptr(), 128, 128, 128, 64, 9, 64 * j, 0, 0, st))
        _lib.check(lib.dmd_pack_conv_weight(w.data_ptr(), pk_lo[j].data_ptr(), 128, 128, 128, 64, 9, 64 * j, 0, 2, st))
    for j in range(8):
        _lib.check(lib.dmd_pack_conv_weight(w.data_ptr(), pk_16[j].data_ptr(), 128, 128, 128, 16, 9, 16 * j, 0, 1, st))
    res = {}
    for S in sizes:
        x = torch.rand(b, S, S, 128, generator=gen).mul(2).sub(1).to(dev)
        hi = torch.empty(lib.dmd_plc16_bytes(b, S, S, 128), dtype=torch.uint8, device=dev)
        lo = torch.empty_like(hi)
        plane = lib.dmd_plc16_bytes(b, S, S, 16) // 2   # one PLC16 plane: 8 channels
        pd = _lib.PrepDesc(src0=x.data_ptr(), C0=128, B=b, Hs=S, Ws=S, eps=1e-5, dst0=hi.data_ptr(), dst_lo0=lo.data_ptr())
        _lib.check(lib.dmd_prep_act(C.byref(pd), st))
        outs = {"three_pass_64": torch.empty(b, S, S, 128, device=dev), "one_launch_16": torch.empty(b, S, S, 128, device=dev)}

        def launch(out, src, src_lo, C0, wpk, precise, first):
            d = _lib.ConvDesc(src0=src, src0_lo=src_lo, C0=C0, B=b, H=S, W=S, taps=9, stride=1, wpk=wpk,
                              bias=bias.data_ptr() if first else None, Cout=128, CoutPad=128,
                              residual=None if first else out.data_ptr(), out=out.data_ptr(), out_gs=32, precise=precise)
            _lib.check(lib.dmd_conv2d_fprop(C.byref(d), st))

        def three_pass():
            o = outs["three_pass_64"]
            for j in range(2):
                off = (64 * j // 8) * plane
                launch(o, hi.data_ptr() + off, None, 64, pk_hi[j].data_ptr(), 0, j == 0)
                launch(o, lo.data_ptr() + off, None, 64, pk_hi[j].data_ptr(), 0, False)
                launch(o, hi.data_ptr() + off, None, 64, pk_lo[j].data_ptr(), 0, False)

        def one_launch():
            o = outs["one_launch_16"]
            for j in range(8):
                off = (16 * j // 8) * plane
                launch(o, hi.data_ptr() + off, lo.data_ptr() + off, 16, pk_16[j].data_ptr(), 1, j == 0)
        three_pass(); one_launch()
        ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
        err = {k: float((o.double() - ref).norm() / ref.norm()) for k, o in outs.items()}
        row = {"error_vs_float64": err}
        for k, fn in (("three_pass_64", three_pass), ("one_launch_16", one_launch)):
            ks = _profile(fn, reps)
            convs = [us for n, _, us in ks if "conv_tc_kernel" in n]
            row[k] = {"launches": len(convs) // reps, "conv_us": sum(convs) / reps}
        res[f"B={b} {S}x{S}"] = row
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["64,128,128,128", "128,128,128,128"])
    ap.add_argument("--envs", type=int, default=32)
    ap.add_argument("--horizon", type=int, default=15)
    ap.add_argument("--reps", type=int, default=10, help="timed repetitions of the policy-only measurements")
    ap.add_argument("--updates", type=int, default=5, help="timed whole cfg-3 updates per round")
    ap.add_argument("--whole-repeats", type=int, default=3, help="rounds of whole cfg-3 updates, alternating the policies")
    ap.add_argument("--trace", action="store_true", help="torch.profiler kernel traces instead of the timings: one forward and "
                    "backward node of --trace-config, and one 128 -> 128 conv in both K-split policies")
    ap.add_argument("--trace-config", default="128,128,128,128")
    ap.add_argument("--dump-outputs", metavar="DIR")
    ap.add_argument("--lib", help="load this build of libdiamond_b200.so instead of the in-tree one")
    args = ap.parse_args()
    import torch

    from diamond_b200 import _lib

    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA GPU")
    dev = torch.device("cuda:0")
    if args.dump_outputs:
        print(json.dumps(dump_outputs(args.dump_outputs, dev)))
        return
    res = {"gpu_before": gpu_state(), "envs": args.envs, "horizon": args.horizon, "torch": torch.__version__}
    if args.trace:
        res["trace"] = {"policy " + args.trace_config: trace_policy([int(x) for x in args.trace_config.split(",")], args.envs, args.reps, dev),
                        "chunk_policies": trace_chunk_policies(args.envs, (64, 32, 16, 8), args.reps, dev)}
    else:
        acs, res["configs"] = [], []
        for c in args.configs:
            ac, out = bench_config([int(x) for x in c.split(",")], args, dev)
            acs.append(ac); res["configs"].append(out)
        whole_updates(acs, res["configs"], args, dev)
    res["gpu_after"] = gpu_state()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
