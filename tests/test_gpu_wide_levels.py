"""GPU: inference with 128-channel U-Net / encoder levels.

- SelfAttention2d at C = 128 (attn_cluster_kernel at L = 64, attn_qkv_kernel + attn_stream_kernel at any other L) against float64,
  output pre-filled with NaN, statistics added to a pre-filled buffer.
- A [64, 128, 128, 128] denoiser (K-split 128 -> 128 convs, 256-channel up-path concats, 256 -> 128 skip projections run as their
  own launches, mid-block attention at C = 128): model output and Euler sample() against the reference's own outputs
  (tests/golden/denoiser_wide.npz, oracle/make_golden_wide.py), and model output against the float64 oracle with a NaN-filled
  workspace.
- A [128] * 4 reward / termination model against the reference (tests/golden/rew_end_wide.npz).
- Training of two such denoisers (one at batch 32) and a reward / termination model against float64 autograd, with the bounds
  of the fp16-operand emulation (oracle/fp16_emulation.py grad_errors)."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

GN_EPS = 1e-5
REL_TOL = 1e-3


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _gn_stats(x, gs):
    b, c = x.shape[0], x.shape[-1]
    v = x.double().reshape(b, -1, c // gs, gs)
    return torch.stack([v.sum(dim=(1, 3)), v.pow(2).sum(dim=(1, 3))], dim=-1).contiguous()


def _ref_attn(x, h, w, gs, gamma, beta, wqkv, bqkv, wout, bout):
    """blocks.py:62-72 in float64 over NHWC x [B][L][C] with L = h * w."""
    b, L, c = x.shape
    xd = x.double().cpu().reshape(b, h, w, c).permute(0, 3, 1, 2)
    y = F.group_norm(xd, c // gs, gamma.double().cpu(), beta.double().cpu(), eps=GN_EPS)
    qkv = F.conv2d(y, wqkv.double().cpu().view(3 * c, c, 1, 1), bqkv.double().cpu())
    nh = c // 8
    qkv = qkv.view(b, nh * 3, 8, L).transpose(2, 3)
    q, k, v = qkv.chunk(3, dim=1)
    att = torch.softmax((q @ k.transpose(-2, -1)) / math.sqrt(8), dim=-1)
    a = (att @ v).transpose(2, 3).reshape(b, c, h, w)
    out = y + F.conv2d(a, wout.double().cpu().view(c, c, 1, 1), bout.double().cpu())
    return out.permute(0, 2, 3, 1).reshape(b, L, c)


@pytest.mark.parametrize("h,w,b", [(8, 8, 3), (8, 8, 132), (11, 11, 5), (19, 35, 4)], ids=["L64", "L64-b132", "L121", "L665"])
def test_attn_fwd_c128(h, w, b):
    from diamond_b200 import _lib

    dev = _dev()
    c, gs, L = 128, 32, h * w
    g = torch.Generator().manual_seed(1000 + L + b)
    n = torch.arange(b, dtype=torch.float32).view(b, 1, 1)
    x = torch.randn(b, L, c, generator=g) * (0.8 + torch.remainder(0.37 * n, 1.0)) + torch.sin(1.7 * n)
    wt = lambda *s: torch.randn(*s, generator=g) / math.sqrt(s[-1])  # noqa: E731
    params = [1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g), wt(3 * c, c), 0.1 * torch.randn(3 * c, generator=g),
              wt(c, c), 0.1 * torch.randn(c, generator=g)]
    ref = _ref_attn(x, h, w, gs, *params)
    x, params = x.to(dev), [p.to(dev) for p in params]
    out = torch.full_like(x, math.nan)
    pre = torch.randn(b, c // gs, 2, generator=g, dtype=torch.float64).to(dev) * 100
    st = pre.clone()
    nbytes = _lib.lib().dmd_attn_scratch_bytes(b, L, c)
    assert (nbytes == 0) == (L == 64)
    scratch = torch.full((max(nbytes, 16) // 4,), math.nan, device=dev)
    _lib.check(_lib.lib().dmd_attn_fwd_scratch(x.data_ptr(), _gn_stats(x, gs).data_ptr(), *[p.data_ptr() for p in params], out.data_ptr(),
                                               st.data_ptr(), b, L, c, gs, GN_EPS, scratch.data_ptr(), nbytes, _lib.current_stream()))
    torch.cuda.synchronize()
    e_out = _rel(out, ref)
    e_st = _rel(st - pre, _gn_stats(ref, gs))
    print(f"attn C=128 L={L} B={b}: out {e_out:.2e} stats {e_st:.2e}")
    assert e_out < 1e-5 and e_st < 1e-5, (e_out, e_st)


def _golden_denoiser(dev):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig
    from oracle import torch_oracle as O
    from oracle.make_golden_wide import DENOISER_WIDE as c

    inner = c["inner"]
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels, list(inner.depths),
                                                   list(inner.channels), list(inner.attn_depths), inner.num_actions), 0.5, 0.3))
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    den.inner_model.load_state_dict(sd)
    return den.to(dev).eval(), sd, c


def test_wide_denoiser_matches_reference_golden(golden_dir):
    from oracle import torch_oracle as O

    dev = _dev()
    den, sd, c = _golden_denoiser(dev)
    g = np.load(os.path.join(golden_dir, "denoiser_wide.npz"))
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    obs, act, x_noisy = O.synthetic_inputs(c["b"], c["inner"], c["h"], c["w"], c["iseed"])
    b, t, ch, h, w = obs.shape
    sig = torch.from_numpy(g["sigmas_in"])
    model, dn = den._native_forward(x_noisy.to(dev), sig.to(dev), obs.reshape(b, t * ch, h, w).to(dev), act.to(dev), True, True)
    err = _rel(model, torch.from_numpy(g["model_output"]))
    diff = (dn.cpu() - torch.from_numpy(g["denoised"])).abs()
    print(f"denoiser_wide: model_output rel L2 {err:.3e}, denoised pixels one level off {float((diff > 0).float().mean()):.3%}")
    assert err < REL_TOL, err
    assert float(diff.max()) <= 2 / 255 + 1e-6 and float((diff > 0).float().mean()) < 0.05


@pytest.mark.parametrize("graph", [False, True])
def test_wide_sampler_matches_reference_golden(golden_dir, graph):
    from diamond_b200.models.diffusion import DiffusionSampler, DiffusionSamplerConfig
    from oracle import torch_oracle as O

    dev = _dev()
    den, _, c = _golden_denoiser(dev)
    g = np.load(os.path.join(golden_dir, "denoiser_wide.npz"))
    s = c["sampler"]
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(s.num_steps_denoising, s.sigma_min, s.sigma_max, s.rho, s.order,
                                                           s.s_churn, s.s_tmin, s.s_tmax, s.s_noise))
    sampler.use_cuda_graph = graph
    assert torch.equal(sampler.sigmas.cpu(), torch.from_numpy(g["sampler_sigmas"]))
    obs, act, _ = O.synthetic_inputs(c["b"], c["inner"], c["h"], c["w"], c["iseed"])
    x0 = torch.from_numpy(g["x0"]).to(dev)
    orig = torch.randn
    torch.randn = lambda *a, **k: x0.clone()   # the reference's draw (Euler without churn draws only x0)
    try:
        for _ in range(2 if graph else 1):     # the second call replays the captured graph
            x, traj = sampler.sample(obs.to(dev), act.to(dev))
    finally:
        torch.randn = orig
    ref, got = torch.from_numpy(g["trajectory"]), torch.stack(traj).cpu()
    assert got.shape == ref.shape and torch.equal(x.cpu(), got[-1])
    diff = (got - ref).abs()
    frac = float((diff > 1e-3).float().mean())
    print(f"denoiser_wide sample (graph={graph}): max|diff| {float(diff.max()):.3e}, frac > 1e-3 {frac:.3e}")
    # a one-level flip of denoised (2/255) moves x by at most 2/255 per Euler step (tests/test_gpu_denoiser.py)
    assert float(diff.max()) <= 3 * 2 / 255 + 1e-5 and frac < 0.08


@pytest.mark.parametrize("channels", [[64, 128, 128, 128], [128, 128, 128, 128]], ids=["64-128-128-128", "128x4"])
def test_wide_denoiser_vs_float64_on_poisoned_workspace(channels):
    """The whole U-Net against the float64 oracle at fresh inputs, with the workspace filled with NaN first: every K-split
    chunk, projection and attention output is written before it is read.  [128] * 4 adds K-split convs and 256-channel
    concats at full resolution, conv_in into and norm_out / conv_out over 128 channels."""
    from diamond_b200 import _lib
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig
    from oracle import torch_oracle as O

    dev = _dev()
    inner = O.InnerCfg(depths=[1, 1, 1, 1], channels=channels)
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels, list(inner.depths),
                                                   list(inner.channels), list(inner.attn_depths), inner.num_actions), 0.5, 0.3))
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), 2469)
    den.inner_model.load_state_dict(sd)
    den = den.to(dev).eval()
    obs, act, x_noisy = O.synthetic_inputs(3, inner, 64, 64, 123)
    b, t, ch, h, w = obs.shape
    sig = torch.tensor([0.3, 1.5, 6.0])
    den.inner_model.workspace(_lib.lib().dmd_denoiser_workspace_bytes(den.inner_model.native(), b, h, w)).fill_(0xFF)   # fp32 NaN
    sd64 = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        ref = O.model_output(x_noisy.double(), sig.double(), obs.reshape(b, t * ch, h, w).double(), act, sd64, O.DenoiserCfg(inner=inner))
    model, _ = den._native_forward(x_noisy.to(dev), sig.to(dev), obs.reshape(b, t * ch, h, w).to(dev), act.to(dev), True, False)
    err = _rel(model, ref)
    print(f"{channels} vs float64: model_output rel L2 {err:.3e}")
    assert torch.isfinite(model).all() and err < REL_TOL, err


def test_wide_rew_end_matches_reference_golden(golden_dir):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from oracle import torch_oracle as O
    from oracle.make_golden_wide import REW_END_WIDE as c

    dev = _dev()
    g = np.load(os.path.join(golden_dir, "rew_end_wide.npz"))
    cfg = c["cfg"]
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    m = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths), list(cfg.channels),
                                      list(cfg.attn_depths), cfg.num_actions))
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    frames, act = torch.from_numpy(g["frames"]).to(dev), torch.from_numpy(g["act"]).to(dev)
    with torch.no_grad():   # the inference entry point, as WorldModelEnv calls it (training is checked below)
        lr, le, hc = m.predict_rew_end(frames[:, 0:3], act[:, 0:3], frames[:, 1:4])
        e = [_rel(torch.cat((lr, le), -1), torch.from_numpy(np.concatenate((g["burn_rew"], g["burn_end"]), -1)))]
        lr, le, hc = m.predict_rew_end(frames[:, 3:4], act[:, 3:4], frames[:, 4:5], hc)
    e += [_rel(torch.cat((lr, le), -1), torch.from_numpy(np.concatenate((g["step3_rew"], g["step3_end"]), -1)))]
    e += [_rel(hc[0], torch.from_numpy(g["hx"])), _rel(hc[1], torch.from_numpy(g["cx"]))]
    print("rew_end_wide rel errors (burn logits, step logits, hx, cx):", ["%.2e" % v for v in e])
    # the bounds of tests/test_gpu_rew_end.py, over each call's 5 head outputs together: the step's 4 end logits alone have an
    # rms of 0.036 (0.17 in that test's fixture), so their own relative error magnifies an absolute error the rest share
    assert max(e) < 2e-3 and max(e[-2:]) < 1e-3, e


# training cases in the shape of oracle/training_configs.py, checked by tests/test_gpu_training_configs.py's float64-autograd
# check with the fp16-operand emulation's bounds (whole gradient within 1.25x of it, each tensor within 2x)
WIDE_TRAINING_CASES = {
    # 128 -> 128 K-split convs and dgrads, 256-channel up-path concats, a 64 -> 128 projection and 256 -> 128 / 192 -> 64 ones
    # as their own launches, stride-2 and upsample convs at 128, attention backward at C = 128; batch 32
    "W1": ("DENOISER_CASES", dict(inner=dict(depths=[1, 1, 1], channels=[64, 128, 128], attn_depths=[0, 0, 0]),
                                  h=32, w=32, b=32, seq=1, mask_off=[], wseed=671, dseed=681)),
    # a 128-channel level 0: conv_in into 128 channels, norm_out / conv_out over 128, 256-channel concats at full resolution
    "W2": ("DENOISER_CASES", dict(inner=dict(cond_channels=64, depths=[1, 1], channels=[128, 128], attn_depths=[0, 1]),
                                  h=16, w=16, b=3, seq=1, mask_off=[], wseed=672, dseed=682)),
    # reward / termination encoder with 128-channel levels and its two attention blocks at C = 128
    "RW": ("REW_END_CASES", dict(cfg=dict(cond_channels=64, img_size=32, depths=[1, 1, 1], channels=[64, 128, 128], attn_depths=[0, 0, 0]),
                                 b=4, T=4, death=(1, 2), pad=(2, 3), wseed=673, dseed=683)),
}


@pytest.mark.parametrize("name", list(WIDE_TRAINING_CASES))
def test_wide_training_matches_float64_autograd(name, monkeypatch):
    import oracle.training_configs as TC
    from oracle import torch_oracle as O

    import importlib.util

    spec = importlib.util.spec_from_file_location("_training_configs_check", os.path.join(os.path.dirname(__file__), "test_gpu_training_configs.py"))
    T = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(T)
    dev = _dev()
    table, c = WIDE_TRAINING_CASES[name]
    c = dict(c)
    if "inner" in c:
        c["inner"] = O.InnerCfg(**c["inner"])
    else:
        c["cfg"] = O.RewEndCfg(**c["cfg"])
    monkeypatch.setitem(getattr(TC, table), name, c)
    T._check_case(name, dev)
