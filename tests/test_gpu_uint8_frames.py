"""GPU: uint8 frame batches (diamond_b200/frames.py) compute what their fp32 decoding computes.

* the packed conv_in operand of the denoiser and the encoder input of the reward/termination model, from uint8 sources
  (all 256 levels x 3 kinds, strided context views), are bit-identical to the fp32 path's;
* Denoiser.forward / RewEndModel.forward on a uint8 batch give the loss, logits and every gradient of the fp32 batch that
  decodes each frame by its kind, within the fp32 path's own run-to-run difference (GroupNorm statistics accumulate with fp64
  atomics, DESIGN.md section 2, so the last bit may move between two runs of either path);
* WorldModelEnv with a uint8 loader: same ring and burn-in state after reset, same frames over 15 steps with deaths, a
  quarter of the pool memory.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import torch_oracle as O

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _maxdiff(a, b) -> float:
    return float((a.double() - b.double()).abs().max()) if a.numel() else 0.0


def _denoiser(dev, b_depths=(2, 2, 2, 2)):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.synthetic import randomize_module_

    inner = O.InnerCfg(depths=list(b_depths))
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths),
                                                   inner.num_actions), 0.5, 0.3))
    randomize_module_(den.inner_model, 3)
    den = den.to(dev).train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    return den, inner


def _rew_end(dev):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import randomize_module_

    c = O.RewEndCfg()
    m = RewEndModel(RewEndModelConfig(c.lstm_dim, c.img_channels, c.img_size, c.cond_channels, list(c.depths), list(c.channels),
                                      list(c.attn_depths), c.num_actions))
    randomize_module_(m, 4)
    return m.to(dev).train(), c


def _find(ws: torch.Tensor, want: torch.Tensor) -> int:
    """Float offset of `want` (flat) inside the workspace `ws` (uint8) -- where the pack kernel wrote its operand."""
    f = ws[: ws.numel() // 4 * 4].view(torch.float32)
    w = want.reshape(-1)
    j = int(w.abs().argmax())   # a random noisy value: few places in the workspace hold it
    for at in (f == w[j]).nonzero().flatten().tolist()[:4096]:
        off = at - j
        if 0 <= off and off + w.numel() <= f.numel() and torch.equal(f[off:off + w.numel()], w):
            return off
    raise AssertionError("the fp32 operand was not found in the workspace")


def test_decode_rows_on_the_gpu():
    """Row 2 (torch's decode on the GPU) against row 1 (Episode.load on the CPU): record how many levels differ."""
    dev = _dev()
    from diamond_b200 import frames as F

    t = F.decode_table(dev).cpu()
    u = torch.arange(256, dtype=torch.uint8)
    assert torch.equal(t[1], u.div(255).mul(2).sub(1))
    assert torch.equal(t[2], u.to(dev).div(255).mul(2).sub(1).cpu())
    assert torch.equal(t[0], torch.zeros(256))
    n = int((t[1] != t[2]).sum())
    print(f"levels where the GPU decode differs from the CPU decode: {n} of 256")
    levels, kinds = F.encode(t[2].to(dev).view(1, 1, 256, 1).expand(1, 3, 256, 1).contiguous())
    assert torch.equal(levels.cpu()[0, 0, :, 0], u) and int(kinds) in (F.KIND_CPU, F.KIND_GPU)
    if n:
        assert int(kinds) == F.KIND_GPU


def _all_levels(b, t, c, h, w, seed):
    """levels (b, t, c, h, w) in which every frame holds all 256 levels; kinds cycling over 0, 1, 2 (and one 7, read as 0)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.arange(c * h * w) % 256
    levels = torch.stack([base[torch.randperm(c * h * w, generator=g)] for _ in range(b * t)]).to(torch.uint8).view(b, t, c, h, w)
    kinds = (torch.arange(b * t) % 3).to(torch.uint8).view(b, t)
    kinds[0, 0] = 7
    return levels, kinds


def test_denoiser_pack_is_bit_identical_to_fp32():
    dev = _dev()
    from diamond_b200 import frames as F

    den, inner = _denoiser(dev, (1, 1, 1, 1))
    im = den.inner_model
    n, c, hw = inner.num_steps_conditioning, inner.img_channels, 64
    b = 6
    levels, kinds = _all_levels(b, n + 2, c, hw, hw, 0)
    levels, kinds = levels.to(dev), kinds.to(dev)
    g = torch.Generator().manual_seed(1)
    noisy = torch.randn(b, c, hw, hw, generator=g).to(dev)
    c_noise = torch.randn(b, generator=g).to(dev)
    act = torch.randint(0, inner.num_actions, (b, n), generator=g).to(dev)
    for i in (0, 1, 2):   # context views frames[:, i:i+n] of the (b, n+2) batch, read in place
        obs_f = (F.decode(levels[:, i:i + n], kinds[:, i:i + n]) / den.cfg.sigma_data).reshape(b, n * c, hw, hw)
        with torch.no_grad():
            im(noisy, c_noise, obs_f, act)
            ws = im._ws
            cp = (n + 1) * c + (-(n + 1) * c) % 8
            want = torch.zeros(b, hw, hw, cp, device=dev)
            want[..., :n * c] = obs_f.permute(0, 2, 3, 1)
            want[..., n * c:(n + 1) * c] = noisy.permute(0, 2, 3, 1)
            off = _find(ws, want)
            f32 = ws.view(torch.float32)[off:off + want.numel()].clone()
            ws.view(torch.float32)[off:off + want.numel()].fill_(float("nan"))
            im(noisy, c_noise, F.U8FrameStack(levels[:, i:i + n], kinds[:, i:i + n], F.context_table(dev, den.cfg.sigma_data)), act)
            assert im._ws.data_ptr() == ws.data_ptr()
            u8 = ws.view(torch.float32)[off:off + want.numel()]
        assert torch.equal(u8, f32), f"context view {i}: the uint8 pack differs from the fp32 pack"


def test_rew_end_pack_is_bit_identical_to_fp32():
    dev = _dev()
    from diamond_b200 import frames as F

    model, c = _rew_end(dev)
    b, t = 4, 5
    levels, kinds = _all_levels(b, t + 1, c.img_channels, c.img_size, c.img_size, 2)
    levels, kinds = levels.to(dev), kinds.to(dev)
    act = torch.randint(0, c.num_actions, (b, t), device=dev)
    fl = F.decode(levels, kinds)
    with torch.no_grad():
        model._predict(fl[:, :-1], act, fl[:, 1:])
        ws = model._ws
        hw = c.img_size * c.img_size
        rows = []
        for k in range(t):
            for n in range(b):
                rows.append(torch.cat([fl[n, k].reshape(c.img_channels, hw), fl[n, k + 1].reshape(c.img_channels, hw)]).t())
        x = torch.stack(rows)   # (t*b, hw, 2C), time-major like the kernel
        for cp in (8, 16):
            want = torch.zeros(t * b, hw, cp, device=dev)
            want[..., :2 * c.img_channels] = x
            try:
                off = _find(ws, want)
                break
            except AssertionError:
                continue
        else:
            raise AssertionError("encoder input not found")
        f32 = ws.view(torch.float32)[off:off + want.numel()].clone()
        ws.view(torch.float32)[off:off + want.numel()].fill_(float("nan"))
        model._predict(levels[:, :-1], act, levels[:, 1:], kinds=(kinds[:, :-1], kinds[:, 1:]))
        assert model._ws.data_ptr() == ws.data_ptr()
        assert torch.equal(ws.view(torch.float32)[off:off + want.numel()], f32)


# ------------------------------------------------------------------------------------------------ denoiser training
def _seg_batch(b, t, c, hw, num_actions, seed, dev):
    """uint8 segments with left-padded (row 0), right-padded (row 1: the last target) and mid-target-padded (row 2) rows;
    padded frames hold random bytes, which must not matter."""
    rng = np.random.default_rng(seed)
    levels = torch.from_numpy(rng.integers(0, 256, size=(b, t, c, hw, hw), dtype=np.uint8))
    act = torch.from_numpy(rng.integers(0, num_actions, size=(b, t)).astype(np.int64))
    mask = torch.ones(b, t, dtype=torch.bool)
    mask[0, :2] = False
    mask[1, t - 1:] = False
    if b > 2:
        mask[2, t - 2:] = False
    return levels.to(dev), act.to(dev), mask.to(dev)


def _den_step(den, obs, act, mask, seed):
    torch.manual_seed(seed)
    den.zero_grad(set_to_none=True)
    loss, _ = den(SimpleNamespace(obs=obs, act=act, mask_padding=mask))
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), [p.grad.detach().clone() for p in den.inner_model.parameters()]


RUNS = 3   # runs of each path: the run-to-run spread is the largest difference over the pairs within a path
# The packed inputs are bit-identical (the two tests above), so any difference comes from the order of the fp64 atomics, which
# follows kernel timing -- and the uint8 pack kernel runs for a different time than the fp32 one.  Measured on the H100, the
# closest cross pair stays within 1.4x the within-path spread; the bound allows 2x.
SPREAD_FACTOR = 2.0


def _assert_within_run_to_run(label, u8_runs, f32_runs):
    """uint8 vs fp32, per tensor: the closest pair of runs across the two paths differs by no more than SPREAD_FACTOR times
    what the runs within a path differ by (every run moves the last bits)."""
    def check(name, us, fs):
        cross = min(_maxdiff(u, f) for u in us for f in fs)
        within = max(_maxdiff(x[i], x[j]) for x in (us, fs) for i in range(len(x)) for j in range(i + 1, len(x)))
        assert cross <= SPREAD_FACTOR * within, f"{label}: {name}: uint8 vs fp32 {cross:.3e}, run-to-run {within:.3e}"
    lu, lf = [r[0] for r in u8_runs], [r[0] for r in f32_runs]
    gu, gf = [r[1] for r in u8_runs], [r[1] for r in f32_runs]
    exact = torch.equal(lu[0], lf[0]) and all(torch.equal(a, b) for a, b in zip(gu[0], gf[0]))
    fp32_exact = torch.equal(lf[0], lf[1]) and all(torch.equal(a, b) for a, b in zip(gf[0], gf[1]))
    print(f"{label}: {len(gf[0])} tensors; uint8 vs fp32 bit-identical: {exact} (fp32 vs fp32: {fp32_exact}); "
          f"loss {float(lu[0]):.7f} vs {float(lf[0]):.7f}")
    check("loss", lu, lf)
    for k in range(len(gf[0])):
        check(f"tensor {k}", [g[k] for g in gu], [g[k] for g in gf])


@pytest.mark.parametrize("b,steps,depths", [(32, 1, (2, 2, 2, 2)), (32, 2, (2, 2, 2, 2)), (256, 1, (2, 2, 2, 2))])
def test_denoiser_training_uint8_matches_fp32_twin(b, steps, depths):
    dev = _dev()
    from diamond_b200 import frames as F

    den, inner = _denoiser(dev, depths)
    t = inner.num_steps_conditioning + steps
    levels, act, mask = _seg_batch(b, t, inner.img_channels, 64, inner.num_actions, 10 + b + steps, dev)
    twin = F.decode(levels, F.kinds_from_mask(mask, (b, t), dev))
    f32 = [_den_step(den, twin, act, mask, 5) for _ in range(RUNS)]
    u8 = [_den_step(den, levels, act, mask, 5) for _ in range(RUNS)]
    assert len(f32[0][1]) == 235
    _assert_within_run_to_run(f"denoiser B={b} steps={steps}", u8, f32)
    with torch.no_grad():   # the no-grad eval call (test_component)
        torch.manual_seed(6)
        lf, _ = den(SimpleNamespace(obs=twin, act=act, mask_padding=mask))
        torch.manual_seed(6)
        lf2, _ = den(SimpleNamespace(obs=twin, act=act, mask_padding=mask))
        torch.manual_seed(6)
        lu, _ = den(SimpleNamespace(obs=levels, act=act, mask_padding=mask))
        torch.manual_seed(6)
        lu2, _ = den(SimpleNamespace(obs=levels, act=act, mask_padding=mask))
    print(f"no-grad: {float(lu):.6f} vs {float(lf):.6f}")
    assert _maxdiff(lu, lf) <= max(_maxdiff(lf, lf2), _maxdiff(lu, lu2))


# ------------------------------------------------------------------------------------------------ reward / termination training
def _rew_batch(dev, uint8_final: bool, seed=3):
    from diamond_b200 import frames as F

    c = O.RewEndCfg()
    b, T = 32, 19
    rng = np.random.default_rng(seed)
    levels = torch.from_numpy(rng.integers(0, 256, size=(b, T, c.img_channels, c.img_size, c.img_size), dtype=np.uint8)).to(dev)
    act = torch.from_numpy(rng.integers(0, c.num_actions, size=(b, T)).astype(np.int64)).to(dev)
    rew = torch.from_numpy(rng.choice([-1.0, 0.0, 0.0, 1.0], size=(b, T)).astype(np.float32)).to(dev)
    end = torch.zeros(b, T, dtype=torch.long, device=dev)
    mask = torch.ones(b, T, dtype=torch.bool, device=dev)
    end[1, 5] = 1; mask[1, 6:] = False             # dies: float final observation
    end[5, 11] = 1; mask[5, 12:] = False           # dies: uint8 (or float) final observation
    mask[2, 10:] = False                           # runs past its episode's end
    fin = {i: torch.from_numpy(rng.integers(0, 256, size=levels.shape[2:], dtype=np.uint8)).to(dev) for i in (1, 5)}
    fin_f = {i: F.decode(v, torch.tensor(F.KIND_GPU, dtype=torch.uint8, device=dev)) for i, v in fin.items()}
    info_f = [{"final_observation": fin_f[i]} if i in fin else {} for i in range(b)]
    info_u = [{"final_observation": (fin[i] if (uint8_final and i == 5) else fin_f[i])} if i in fin else {} for i in range(b)]
    twin = F.decode(levels, F.kinds_from_mask(mask, (b, T), dev))
    mk = lambda obs, info: SimpleNamespace(obs=obs.clone(), act=act, rew=rew, end=end, trunc=torch.zeros_like(end),
                                           mask_padding=mask, info=info)
    return mk(levels, info_u), mk(twin, info_f)


def _rew_step(model, batch):
    seen = {}
    inner = model.predict_rew_end

    def tap(*a, **k):
        out = inner(*a, **k)
        seen["logits"] = torch.cat([out[0].detach(), out[1].detach()], -1)
        return out
    model.predict_rew_end = tap
    try:
        loss, _ = model(batch)
    finally:
        del model.predict_rew_end
    model.zero_grad(set_to_none=True)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), [seen["logits"]] + [p.grad.detach().clone() for p in model.parameters()]


@pytest.mark.parametrize("uint8_final", [False, True])
def test_rew_end_training_uint8_matches_fp32_twin(uint8_final):
    dev = _dev()
    model, _ = _rew_end(dev)
    bu, bf = _rew_batch(dev, uint8_final)
    f32 = [_rew_step(model, SimpleNamespace(**{**bf.__dict__, "obs": bf.obs.clone()})) for _ in range(RUNS)]
    u8 = [_rew_step(model, SimpleNamespace(**{**bu.__dict__, "obs": bu.obs.clone()})) for _ in range(RUNS)]
    _assert_within_run_to_run(f"rew_end 32x19 uint8 final obs={uint8_final}", u8, f32)


def test_rew_end_off_grid_final_observation_raises():
    dev = _dev()
    model, _ = _rew_end(dev)
    bu, _ = _rew_batch(dev, False)
    bu.info[1]["final_observation"] = bu.info[1]["final_observation"] + 1e-3
    with pytest.raises(ValueError, match="not decoded levels"):
        model(bu)


# ------------------------------------------------------------------------------------------------ WorldModelEnv
def _env(den, rew_end, uint8: bool, dev):
    from diamond_b200 import frames as F
    from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.diffusion import DiffusionSamplerConfig

    class Loader:
        batch_sampler = SimpleNamespace(batch_size=8)

        def __iter__(self):
            rng = np.random.default_rng(0)
            while True:
                levels = torch.from_numpy(rng.integers(0, 256, size=(8, 4, 3, 64, 64), dtype=np.uint8))
                act = torch.from_numpy(rng.integers(0, 4, size=(8, 4)).astype(np.int64))
                if uint8:   # no mask_padding: every frame is real
                    yield SimpleNamespace(obs=levels, act=act)
                else:
                    yield SimpleNamespace(obs=F.cpu_decode(levels), act=act)

    return WorldModelEnv(den, rew_end, Loader(), WorldModelEnvConfig(3, 2, DiffusionSamplerConfig(3)))


def test_world_model_env_with_uint8_loader():
    dev = _dev()
    den, _ = _denoiser(dev, (1, 1, 1, 1))
    den.eval()
    rew_end, _ = _rew_end(dev)
    rew_end.eval()
    for p in rew_end.parameters():
        p.requires_grad_(False)
    runs = {}
    for name, uint8 in (("f32", False), ("u8", True), ("f32b", False)):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        env = _env(den, rew_end, uint8, dev)
        torch.manual_seed(0)
        env.reset()
        pool_bytes = env._pool.obs.numel() * env._pool.obs.element_size()
        state = (env.obs_buffer.clone(), env.hx_rew_end.clone(), env.cx_rew_end.clone())
        frames, deaths = [], 0
        for step in range(15):
            act = torch.randint(0, 4, (8,), device=dev)
            obs, rew, end, trunc, info = env.step(act)
            deaths += int(torch.logical_or(end, trunc).sum())
            frames.append(obs)
        runs[name] = (state, torch.stack(frames), pool_bytes, deaths)
    (s_f, fr_f, pb_f, d_f), (s_u, fr_u, pb_u, _), (s_f2, fr_f2, _, _) = runs["f32"], runs["u8"], runs["f32b"]
    assert d_f >= 8, "the horizon must force deaths"
    assert torch.equal(s_u[0], s_f[0]), "ring after reset"
    for a, b, b2 in zip(s_u[1:], s_f[1:], s_f2[1:]):
        assert _maxdiff(a, b) <= _maxdiff(b, b2), "burn-in (hx, cx)"
    print(f"burn-in state bit-identical: {all(torch.equal(a, b) for a, b in zip(s_u[1:], s_f[1:]))}; "
          f"pool bytes uint8 {pb_u} vs fp32 {pb_f}")
    d = (fr_u - fr_f).abs()
    assert float(d.max()) <= 3 * 2 / 255 + 1e-5
    assert float((d > 1e-3).float().mean()) < 0.08
    assert pb_u * 4 == pb_f
