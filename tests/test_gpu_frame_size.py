"""GPU: frame sizes whose deepest U-Net level is not 8 x 8, so that self-attention runs over other token counts (L != 64):
attn_qkv_kernel + attn_stream_kernel one entry point at a time against float64, the denoiser and the sampler against the
reference's own outputs at 84 x 84 (121 tokens) and 150 x 280 (the CSGO shape of BASELINE cfg 5, 665 tokens), the cfg-5
batch of 8 images against the fp32 oracle, reward / termination inference at 128 x 128 (256 tokens), and the training entry
points' rejection of such plans (the attention backward is built for 64 tokens only)."""
import math
import os

import numpy as np
import pytest
import torch

import test_gpu_denoiser as TD
from oracle.make_golden_frame_size import FRAME_SIZE_CASES, initial_noise, noise_checksum

pytestmark = pytest.mark.gpu

TOL = 1e-5
STATS_TOL = 1e-6
REL_TOL = 1e-3
GN_EPS = 1e-5
ATTN_BWD_MSG = "attention backward"


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.double(), b.double().to(a.device)
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------ attention, one op
def _gn_stats(x, gs):
    """(sum, sumsq) per (image, group) of NHWC-flat x [B][L][C], float64."""
    b, L, c = x.shape
    xg = x.double().reshape(b, L, c // gs, gs)
    return torch.stack((xg.sum(dim=(1, 3)), xg.pow(2).sum(dim=(1, 3))), dim=-1).contiguous()


def ref_attn_tokens(x, gs, gamma, beta, wqkv, bqkv, wout, bout):
    """SelfAttention2d (blocks.py:62-72) over the L tokens of x [B][L][C] in float64, one image and head at a time (at
    L = 4096 the whole score tensor of 8 images would take 8.6 GB)."""
    b, L, c = x.shape
    xg = x.double().reshape(b, L, c // gs, gs)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = xg.var(dim=(1, 3), unbiased=False, keepdim=True)
    xn = ((xg - mean) / torch.sqrt(var + GN_EPS)).reshape(b, L, c) * gamma.double() + beta.double()
    qkv = xn @ wqkv.double().T + bqkv.double()
    y = torch.empty(b, L, c, dtype=torch.float64, device=x.device)
    for n in range(b):
        for h in range(c // 8):
            q, k, v = (qkv[n, :, p * c + 8 * h:p * c + 8 * h + 8] for p in range(3))
            y[n, :, 8 * h:8 * h + 8] = torch.softmax(q @ k.T / math.sqrt(8), dim=-1) @ v
    return xn + y @ wout.double().T + bout.double()


def _attn_inputs(g, b, L, c, dev):
    n = torch.arange(b, dtype=torch.float32).view(b, 1, 1)
    x = torch.randn(b, L, c, generator=g) * (0.8 + torch.remainder(0.37 * n, 1.0)) + torch.sin(1.7 * n)
    w = lambda *s: torch.randn(*s, generator=g) / math.sqrt(s[-1])  # noqa: E731
    ps = (x, 1 + 0.2 * torch.randn(c, generator=g), 0.2 * torch.randn(c, generator=g), w(3 * c, c), 0.1 * torch.randn(3 * c, generator=g),
          w(c, c), 0.1 * torch.randn(c, generator=g))
    return [t.to(dev) for t in ps]


def _attn_scratch_call(params, stats_in, out, st, b, L, c, gs, scratch):
    from diamond_b200 import _lib

    _lib.check(_lib.lib().dmd_attn_fwd_scratch(*[t.data_ptr() for t in (params[0], stats_in)], *[t.data_ptr() for t in params[1:]],
                                               out.data_ptr(), st.data_ptr(), b, L, c, gs, GN_EPS,
                                               scratch.data_ptr() if scratch.numel() else None, scratch.numel() * scratch.element_size(),
                                               _lib.current_stream()))


@pytest.mark.parametrize("b", [1, 3, 8])
@pytest.mark.parametrize("c,gs", [(32, 8), (32, 32), (64, 8), (64, 32), (64, 64)])
@pytest.mark.parametrize("L", [16, 45, 100, 121, 256, 665, 4096])
def test_attn_any_token_count(L, c, gs, b):
    """Output (and scratch) pre-filled with NaN; the statistics are added to a pre-filled buffer and compared with float64
    sums of the output the kernel wrote."""
    dev = _dev()
    from diamond_b200 import _lib

    g = torch.Generator().manual_seed(L * 1000 + c * 10 + gs + b)
    params = _attn_inputs(g, b, L, c, dev)
    ref = ref_attn_tokens(params[0], gs, *params[1:])
    out = torch.full_like(params[0], math.nan)
    pre = torch.randn(b, c // gs, 2, generator=g, dtype=torch.float64).to(dev) * 100
    st = pre.clone()
    nbytes = _lib.lib().dmd_attn_scratch_bytes(b, L, c)
    assert nbytes == b * L * 3 * c * 4
    scratch = torch.full((nbytes // 4,), math.nan, device=dev)
    _attn_scratch_call(params, _gn_stats(params[0], gs), out, st, b, L, c, gs, scratch)
    e_out, e_st = _rel(out, ref), _rel(st - pre, _gn_stats(out, gs))
    print(f"attn L={L} C={c} gs={gs} B={b}: out {e_out:.2e} stats {e_st:.2e}")
    assert e_out < TOL and e_st < STATS_TOL, (e_out, e_st)


@pytest.mark.parametrize("c,gs", [(32, 32), (64, 16), (64, 32)])
def test_attn_scratch_entry_point_at_64_tokens_is_dmd_attn_fwd(c, gs):
    """L = 64 keeps the one-launch kernel: through the new entry point (no scratch) the output and statistics are
    bit-identical to dmd_attn_fwd's."""
    dev = _dev()
    from diamond_b200 import _lib

    b = 5
    params = _attn_inputs(torch.Generator().manual_seed(c + gs), b, 64, c, dev)
    stats_in = _gn_stats(params[0], gs)
    assert _lib.lib().dmd_attn_scratch_bytes(b, 64, c) == 0
    out0, out1 = torch.full_like(params[0], math.nan), torch.full_like(params[0], math.nan)
    st0, st1 = torch.zeros(b, c // gs, 2, dtype=torch.float64, device=dev), torch.zeros(b, c // gs, 2, dtype=torch.float64, device=dev)
    _lib.check(_lib.lib().dmd_attn_fwd(*[t.data_ptr() for t in (params[0], stats_in)], *[t.data_ptr() for t in params[1:]], out0.data_ptr(),
                                       st0.data_ptr(), b, 64, c, gs, GN_EPS, _lib.current_stream()))
    _attn_scratch_call(params, stats_in, out1, st1, b, 64, c, gs, torch.empty(0, device=dev))
    torch.cuda.synchronize()
    assert torch.equal(out0, out1)
    assert torch.allclose(st0, st1, rtol=1e-12, atol=0)   # fp64 atomics commute to the last bit only


# ------------------------------------------------------------------------------------------------ denoiser / sampler vs the reference
@pytest.fixture
def frame_size_cases(monkeypatch):
    """The reference-golden checks of test_gpu_denoiser.py, run on the frame-size fixtures."""
    monkeypatch.setattr(TD, "_cases", lambda: FRAME_SIZE_CASES)


@pytest.mark.parametrize("name", list(FRAME_SIZE_CASES))
def test_denoiser_matches_reference_golden_at_frame_size(golden_dir, name, frame_size_cases):
    TD.test_denoiser_matches_reference_golden(golden_dir, name)


@pytest.mark.parametrize("graph", [False, True])
def test_sampler_84x84_matches_reference_golden(golden_dir, graph, frame_size_cases):
    TD.test_sampler_matches_reference_golden(golden_dir, "denoiser_84x84", graph)


def test_sampler_150x280_ten_euler_steps(golden_dir):
    """cfg-5 shape, 10 Euler steps, through the captured CUDA graph.  (1) The loop arithmetic is exact: the oracle loop with
    the CUDA Denoiser.denoise plugged in reproduces the trajectory.  (2) Against the reference's sample_x: step i moves x by
    (x - D_i) dt_i / sigma_i with |dt_i| <= sigma_i, so a one-level flip of the denoised frame D_i (2/255) moves a pixel by at
    most 2/255, and earlier differences are carried with the factor sigma_{i+1} / sigma_i < 1; the last step (sigma = 0) sets
    x = D_9.  A pixel is thus at most 10 levels away; and as for 3 steps, few pixels differ at all."""
    dev = _dev()
    from diamond_b200.models.diffusion import DiffusionSampler, DiffusionSamplerConfig
    from oracle import torch_oracle as O

    c = FRAME_SIZE_CASES["denoiser_150x280"]
    g = np.load(os.path.join(golden_dir, "denoiser_150x280.npz"))
    den, _ = TD._build(c["inner"], c["wseed"], dev)
    s = c["sampler"]
    sampler = DiffusionSampler(den, DiffusionSamplerConfig(s.num_steps_denoising))
    assert torch.equal(sampler.sigmas.cpu(), torch.from_numpy(g["sampler_sigmas"]))
    obs, act, _ = O.synthetic_inputs(c["b"], c["inner"], c["h"], c["w"], c["iseed"])
    x0 = initial_noise(c)   # the reference's first draw, regenerated (the fixture stores its checksum)
    assert np.allclose(noise_checksum(x0), g["x0_checksum"], rtol=1e-12, atol=0)
    x0 = x0.to(dev)
    orig = torch.randn
    torch.randn = lambda *a, **k: x0.clone()
    try:
        for _ in range(2):   # capture, then replay the graph
            x, traj = sampler.sample(obs.to(dev), act.to(dev))
    finally:
        torch.randn = orig
    got = torch.stack(traj).cpu()
    assert torch.equal(x.cpu(), got[-1])

    def cuda_denoise(x_, s_, o_, a_):
        return den.denoise(x_.to(dev), s_.reshape(-1).to(dev), o_.to(dev), a_.to(dev)).cpu()

    with torch.no_grad():
        _, loop = O.sample(obs, act, x0.cpu(), None, None, s, None, denoise_fn=cuda_denoise)
    d_loop = (got - torch.stack(loop)).abs()
    print(f"150x280 loop arithmetic: max|diff|={float(d_loop.max()):.3e} frac>1e-6={float((d_loop > 1e-6).float().mean()):.3e}")
    assert float((d_loop > 1e-6).float().mean()) < 2e-3, float(d_loop.max())
    diff = (x.cpu() - torch.from_numpy(g["sample_x"])).abs()
    frac = float((diff > 1e-3).float().mean())
    print(f"150x280 sample_x vs reference: max|diff|={float(diff.max()):.3e} frac>1e-3={frac:.3e}")
    assert float(diff.max()) <= s.num_steps_denoising * 2 / 255 + 1e-5
    assert frac < 0.08


def test_cfg5_batch_of_eight_matches_the_oracle():
    """One denoiser forward at the per-GPU batch of cfg 5 (8 images of 150 x 280) against the fp32 oracle (run on the GPU
    with TF32 off), every image within 1e-3 relative L2."""
    dev = _dev()
    from oracle import torch_oracle as O

    inner = O.InnerCfg()
    den, sd = TD._build(inner, 2025, dev)
    cfg = O.DenoiserCfg(inner=inner)
    b = 8
    obs, act, x_noisy = O.synthetic_inputs(b, inner, 150, 280, 4243)
    flat = obs.reshape(b, -1, 150, 280)
    sig = torch.linspace(0.002, 20.0, b)
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = O.model_output(x_noisy.to(dev), sig.to(dev), flat.to(dev), act.to(dev), {k: v.to(dev) for k, v in sd.items()}, cfg)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    model, _ = den._native_forward(x_noisy.to(dev), sig.to(dev), flat.to(dev), act.to(dev), True, False)
    per = [_rel(model[i], ref[i]) for i in range(b)]
    print("cfg-5 B=8 per-image rel L2 err:", ["%.2e" % e for e in per])
    assert max(per) < REL_TOL, per


# ------------------------------------------------------------------------------------------------ reward / termination, rejections
def _rew_end(cfg, sd, dev):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig

    m = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths), list(cfg.channels),
                                      list(cfg.attn_depths), cfg.num_actions))
    m.load_state_dict(sd)
    return m.to(dev)


def test_rew_end_inference_at_128_matches_the_oracle():
    """img_size 128: the encoder's attention blocks run over 16 x 16 = 256 tokens."""
    dev = _dev()
    from oracle import torch_oracle as O

    cfg = O.RewEndCfg(img_size=128)
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 778)
    m = _rew_end(cfg, sd, dev).eval()
    rng = np.random.default_rng(95)
    b, t = 3, 2
    frames = torch.from_numpy(rng.integers(0, 256, size=(b, t + 1, 3, 128, 128)).astype(np.float32)).div(255).mul(2).sub(1)
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, t)).astype(np.int64))
    with torch.no_grad():
        rr, re, (rh, rc) = O.predict_rew_end(frames[:, :t], act, frames[:, 1:], sd, cfg)
        lr, le, (hx, cx) = m.predict_rew_end(frames[:, :t].to(dev), act.to(dev), frames[:, 1:].to(dev))
    e = [_rel(lr.cpu(), rr), _rel(le.cpu(), re), _rel(hx[0].cpu(), rh[0]), _rel(cx[0].cpu(), rc[0])]
    print("rew_end 128x128 rel errors (rew, end, hx, cx):", ["%.2e" % v for v in e])
    assert max(e) < 2e-3 and max(e[2:]) < 1e-3, e   # bounds of test_gpu_rew_end.py


class _DenBatch:
    def __init__(self, obs, act, mask):
        self.obs, self.act, self.mask_padding = obs, act, mask


def test_denoiser_training_at_128_is_rejected_before_any_launch():
    """Denoiser.forward (training) at 128 x 128 (mid-block attention over 16 x 16 tokens) fails with an error naming the
    missing attention backward; the C entry points fail before launching anything.  Inference still runs afterwards."""
    dev = _dev()
    from diamond_b200 import _lib
    from diamond_b200.models.diffusion import SigmaDistributionConfig
    from oracle import torch_oracle as O

    inner = O.InnerCfg(depths=[1, 1, 1, 1])
    den, _ = TD._build(inner, 11, dev)
    den.train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    obs = torch.rand(2, inner.num_steps_conditioning + 1, 3, 128, 128, device=dev) * 2 - 1
    act = torch.randint(0, inner.num_actions, (2, inner.num_steps_conditioning + 1), device=dev)
    with pytest.raises(RuntimeError, match=ATTN_BWD_MSG):
        den(_DenBatch(obs, act, torch.ones(2, inner.num_steps_conditioning + 1, dtype=torch.bool, device=dev)))
    lib = _lib.lib()
    h = den.inner_model.native()
    assert lib.dmd_denoiser_train_workspace_bytes(h, 2, 128, 128) == 0
    assert ATTN_BWD_MSG in lib.dmd_last_error().decode()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    lib.dmd_launch_count(1)
    p = obs.data_ptr()
    rc = lib.dmd_inner_model_forward_train(h, 2, 128, 128, p, p, 0, p, act.data_ptr(), p, ws.data_ptr(), ws.numel(), _lib.current_stream())
    assert rc != 0 and ATTN_BWD_MSG in lib.dmd_last_error().decode()
    assert lib.dmd_launch_count(0) == 0
    # the padded-training rejection is unchanged
    assert lib.dmd_denoiser_train_workspace_bytes(h, 2, 60, 62) == 0 and "pad / crop adjoints" in lib.dmd_last_error().decode()
    den.eval()
    with torch.no_grad():
        x = torch.randn(2, 3, 128, 128, device=dev)
        out = den.denoise(x, torch.full((2,), 1.0, device=dev), obs[:, :-1].reshape(2, -1, 128, 128), act[:, :-1])
    torch.cuda.synchronize()
    assert out.shape == (2, 3, 128, 128) and bool(torch.isfinite(out).all())


class _RewBatch:
    def __init__(self, obs, act, rew, end, mask):
        self.obs, self.act, self.rew, self.end, self.mask_padding = obs, act, rew, end, mask
        self.trunc = torch.zeros_like(end)
        self.info = [{}] * obs.size(0)


def test_rew_end_training_at_128_is_rejected_before_any_launch():
    dev = _dev()
    from diamond_b200 import _lib
    from oracle import torch_oracle as O

    cfg = O.RewEndCfg(img_size=128)
    m = _rew_end(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 779), dev).train()
    b, t = 2, 3
    obs = torch.rand(b, t + 1, 3, 128, 128, device=dev) * 2 - 1
    act = torch.randint(0, cfg.num_actions, (b, t + 1), device=dev)
    batch = _RewBatch(obs, act, torch.zeros(b, t + 1, device=dev), torch.zeros(b, t + 1, dtype=torch.long, device=dev),
                      torch.ones(b, t + 1, dtype=torch.bool, device=dev))
    with pytest.raises(RuntimeError, match=ATTN_BWD_MSG):
        m(batch)
    lib = _lib.lib()
    h = m._native()
    assert lib.dmd_rew_end_train_workspace_bytes(h, b, t) == 0 and ATTN_BWD_MSG in lib.dmd_last_error().decode()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    out = torch.empty(b * t * 8 + 4 * b * cfg.lstm_dim, device=dev)
    lib.dmd_launch_count(1)
    rc = lib.dmd_rew_end_forward_train(h, b, t, obs.data_ptr(), obs.data_ptr(), act.data_ptr(), None, None, *[out.data_ptr()] * 4,
                                       ws.data_ptr(), ws.numel(), _lib.current_stream())
    assert rc != 0 and ATTN_BWD_MSG in lib.dmd_last_error().decode()
    assert lib.dmd_launch_count(0) == 0
    m.eval()
    with torch.no_grad():
        lr, le, _ = m.predict_rew_end(obs[:, :t], act[:, :t], obs[:, 1:])
    torch.cuda.synchronize()
    assert lr.shape == (b, t, 3) and bool(torch.isfinite(lr).all() and torch.isfinite(le).all())
