"""GPU: conditioning vectors wider than 256 channels (cond_channels up to 2048).

- dmd_film_wgrad on its own against float64 at CC from 32 to 2048, batches on both sides of its 64-sample chunk, row counts that
  are not multiples of 8, onto a pre-filled buffer (the op adds); at CC <= 256 it keeps its one-launch (rows / 8) x 1 grid.
- A cond_channels = 2048, [64, 128, 128, 128] denoiser: model output and Euler sample() against the reference's own outputs
  (tests/golden/denoiser_cond2048.npz, oracle/make_golden_cond.py), and the cond_channels = 512 reward / termination model's
  predictions against tests/golden/rew_end_cond512.npz.
- Training against float64 autograd with the fp16-operand emulation's bounds (tests/test_gpu_training_configs.py): the denoiser at
  CC = 2048 over two autoregressive steps, the reward / termination model at CC = 512 and 2048 with a death and a padded tail; a
  uint8 batch against float64 autograd and against its fp32 twin; the batch-256 step of a net whose dcond = dfilm Wf split-K
  partials outgrow the backward temporary and get their own buffer, read from the real plan (dmd_denoiser_train_dcond_plan),
  which also keeps the earlier capped plan at every cond_channels <= 256 net tried.
- *_backward_accumulate = prefill + plain call, and both on poisoned workspaces, at CC = 2048.
- Two autoregressive steps leave one flat buffer whose views are the .grads."""
import importlib.util
import json
import math
import os
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
REL_TOL = 1e-3   # model output, as tests/test_gpu_denoiser.py


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _load(name):
    """A sibling test module by file (its helpers; the module is not a package)."""
    spec = importlib.util.spec_from_file_location(f"_cond_width_{name}", os.path.join(HERE, name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


# ------------------------------------------------------------------------------------------------ dmd_film_wgrad
def _film_case(b, cc, rows, seed):
    g = torch.Generator().manual_seed(seed)
    dfilm, cond = torch.randn(b, rows, generator=g), torch.randn(b, cc, generator=g)
    woff = torch.randperm(rows, generator=g) * cc          # rows scattered over the buffer in shuffled order
    boff = rows * cc + torch.randperm(rows, generator=g)
    n = rows * cc + rows + 3
    pre = torch.randn(n, generator=g)
    return dfilm, cond, woff, boff, pre


def _film_run(dfilm, cond, woff, boff, pre, inv, dev):
    from diamond_b200 import ops

    grads = pre.to(dev).clone()
    ops.film_wgrad(dfilm.to(dev), cond.to(dev), grads, woff.to(dev), boff.to(dev), torch.tensor([inv], device=dev))
    torch.cuda.synchronize()
    return grads.cpu()


@pytest.mark.parametrize("cc", [32, 256, 288, 512, 2048])
@pytest.mark.parametrize("b", [1, 63, 64, 65, 256])
def test_film_wgrad_any_cond_width_against_float64(b, cc):
    dev = _dev()
    rows = 203 if b < 256 else 1029
    dfilm, cond, woff, boff, pre = _film_case(b, cc, rows, 31 * b + cc)
    inv = 0.25
    got = _film_run(dfilm, cond, woff, boff, pre, inv, dev)
    d, c = dfilm.double(), cond.double()
    ref = pre.double().clone()
    ref[(woff[:, None] + torch.arange(cc)).reshape(-1)] += (inv * d.t() @ c).reshape(-1)
    ref[boff] += inv * d.sum(0)
    # each sum is b fp32 fmas in a fixed order: bound the error by the sum of magnitudes
    mag = pre.double().abs().clone()
    mag[(woff[:, None] + torch.arange(cc)).reshape(-1)] += (inv * d.abs().t() @ c.abs()).reshape(-1)
    mag[boff] += inv * d.abs().sum(0)
    err = (got.double() - ref).abs()
    worst = float((err / mag.clamp_min(1e-30)).max())
    print(f"film_wgrad B={b} CC={cc} rows={rows}: worst error / magnitude {worst:.2e}")
    assert torch.isfinite(got).all()
    assert bool((err <= 4e-7 * (b + 2) * mag + 1e-30).all()), worst
    # no slot outside the tables moved
    assert torch.equal(got[-3:], pre[-3:])


def _kernel_launches(fn, dev, repeats=4):
    """(name, grid, block) of the CUDA kernels of `repeats` calls of fn, from a torch.profiler trace.  A trace can miss a short
    kernel's record, so fn runs several times and the caller checks the shape of each record it got."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return [(e["name"], tuple(e["args"].get("grid", ())), tuple(e["args"].get("block", ())))
            for e in events if e.get("cat") == "kernel"]


@pytest.mark.parametrize("cc,grid_y", [(32, 1), (256, 1), (288, 2), (2048, 8)])
def test_film_wgrad_launch_shape(cc, grid_y):
    """One launch per call; at CC <= 256 the grid is (ceil(rows / 8), 1, 1), as before wider conditioning existed; above, one
    grid row per 256-column slice of cond."""
    from diamond_b200 import _lib

    dev = _dev()
    rows, b = 7163, 64
    dfilm, cond, woff, boff, pre = _film_case(b, cc, rows, cc)
    args = [t.to(dev) for t in (dfilm, cond)] + [pre.to(dev).clone()] + [t.to(dev) for t in (woff, boff)]
    inv = torch.tensor([1.0], device=dev)
    from diamond_b200 import ops

    ops.film_wgrad(*args, inv)   # warm-up: module load
    lib = _lib.lib()
    lib.dmd_launch_count(1)
    ops.film_wgrad(*args, inv)
    assert lib.dmd_launch_count(0) == 1
    k = [x for x in _kernel_launches(lambda: ops.film_wgrad(*args, inv), dev) if "film_wgrad" in x[0]]
    print(f"film_wgrad CC={cc}: {k}")
    assert 1 <= len(k) <= 4   # the launch count per call is pinned above
    for name, grid, block in k:
        assert grid == ((rows + 7) // 8, grid_y, 1) and block == (256, 1, 1), (grid, block)


# ------------------------------------------------------------------------------------------------ inference vs the reference
def _golden_denoiser(dev):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig
    from oracle import torch_oracle as O
    from oracle.make_golden_cond import DENOISER_COND as c

    inner = c["inner"]
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels, list(inner.depths),
                                                   list(inner.channels), list(inner.attn_depths), inner.num_actions), 0.5, 0.3))
    sd = O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"])
    den.inner_model.load_state_dict(sd)
    return den.to(dev).eval(), sd, c


def test_cond2048_denoiser_matches_reference_golden(golden_dir):
    from oracle import torch_oracle as O

    dev = _dev()
    den, sd, c = _golden_denoiser(dev)
    g = np.load(os.path.join(golden_dir, "denoiser_cond2048.npz"))
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    obs, act, x_noisy = O.synthetic_inputs(c["b"], c["inner"], c["h"], c["w"], c["iseed"])
    b, t, ch, h, w = obs.shape
    sig = torch.from_numpy(g["sigmas_in"])
    model, dn = den._native_forward(x_noisy.to(dev), sig.to(dev), obs.reshape(b, t * ch, h, w).to(dev), act.to(dev), True, True)
    err = _rel(model, torch.from_numpy(g["model_output"]))
    diff = (dn.cpu() - torch.from_numpy(g["denoised"])).abs()
    print(f"denoiser_cond2048: model_output rel L2 {err:.3e}, denoised pixels one level off {float((diff > 0).float().mean()):.3%}")
    assert err < REL_TOL, err
    assert float(diff.max()) <= 2 / 255 + 1e-6 and float((diff > 0).float().mean()) < 0.05


@pytest.mark.parametrize("graph", [False, True])
def test_cond2048_sampler_matches_reference_golden(golden_dir, graph):
    from diamond_b200.models.diffusion import DiffusionSampler, DiffusionSamplerConfig
    from oracle import torch_oracle as O

    dev = _dev()
    den, _, c = _golden_denoiser(dev)
    g = np.load(os.path.join(golden_dir, "denoiser_cond2048.npz"))
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
    print(f"denoiser_cond2048 sample (graph={graph}): max|diff| {float(diff.max()):.3e}, frac > 1e-3 {frac:.3e}")
    # a one-level flip of denoised (2/255) moves x by at most 2/255 per Euler step (tests/test_gpu_denoiser.py)
    assert float(diff.max()) <= 3 * 2 / 255 + 1e-5 and frac < 0.08


def test_cond512_rew_end_matches_reference_golden(golden_dir):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from oracle import torch_oracle as O
    from oracle.make_golden_cond import REW_END_COND as c

    dev = _dev()
    g = np.load(os.path.join(golden_dir, "rew_end_cond512.npz"))
    cfg = c["cfg"]
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), c["wseed"])
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    m = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths), list(cfg.channels),
                                      list(cfg.attn_depths), cfg.num_actions))
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    frames, act = torch.from_numpy(g["frames"]).to(dev), torch.from_numpy(g["act"]).to(dev)
    with torch.no_grad():
        lr, le, hc = m.predict_rew_end(frames[:, 0:3], act[:, 0:3], frames[:, 1:4])
        e = [_rel(torch.cat((lr, le), -1), torch.from_numpy(np.concatenate((g["burn_rew"], g["burn_end"]), -1)))]
        lr, le, hc = m.predict_rew_end(frames[:, 3:4], act[:, 3:4], frames[:, 4:5], hc)
    e += [_rel(torch.cat((lr, le), -1), torch.from_numpy(np.concatenate((g["step3_rew"], g["step3_end"]), -1)))]
    e += [_rel(hc[0], torch.from_numpy(g["hx"])), _rel(hc[1], torch.from_numpy(g["cx"]))]
    print("rew_end_cond512 rel errors (burn logits, step logits, hx, cx):", ["%.2e" % v for v in e])
    assert max(e) < 2e-3 and max(e[-2:]) < 1e-3, e   # the bounds of tests/test_gpu_wide_levels.py


# ------------------------------------------------------------------------------------------------ training vs float64
# cases in the shape of oracle/training_configs.py, checked by tests/test_gpu_training_configs.py's float64-autograd check with
# the fp16-operand emulation's bounds (whole gradient within 1.25x of it, each tensor within 2x)
COND_TRAINING_CASES = {
    # a 2048-wide conditioning path over two autoregressive steps, one padded target; 32 / 64 / 128-channel levels
    "C1": ("DENOISER_CASES", dict(inner=dict(cond_channels=2048, depths=[1, 1, 1], channels=[32, 64, 128], attn_depths=[0, 0, 0]),
                                  h=32, w=32, b=2, seq=2, mask_off=[(1, 5)], wseed=691, dseed=692)),
    # the default encoder at cond 512: FiLM rows read act_emb(act) directly
    "RC1": ("REW_END_CASES", dict(cfg=dict(cond_channels=512), b=4, T=7, death=(1, 3), pad=(2, 5), wseed=693, dseed=694)),
    # cond 2048 with attention at C = 32 in the last level, 18 actions
    "RC2": ("REW_END_CASES", dict(cfg=dict(lstm_dim=256, img_channels=1, img_size=32, cond_channels=2048, depths=[1, 2, 1],
                                           channels=[64, 64, 32], attn_depths=[0, 0, 1], num_actions=18),
                                  b=5, T=4, death=(3, 1), pad=(0, 2), wseed=695, dseed=696)),
}


def _case(name):
    from oracle import torch_oracle as O

    table, c = COND_TRAINING_CASES[name]
    c = dict(c)
    if "inner" in c:
        c["inner"] = O.InnerCfg(**c["inner"])
    else:
        c["cfg"] = O.RewEndCfg(**c["cfg"])
    return table, c


@pytest.mark.parametrize("name", list(COND_TRAINING_CASES))
def test_cond_width_training_matches_float64_autograd(name, monkeypatch):
    import oracle.training_configs as TC

    T = _load("test_gpu_training_configs")
    dev = _dev()
    table, c = _case(name)
    monkeypatch.setitem(getattr(TC, table), name, c)
    T._check_case(name, dev)


def _den_step(den, obs, act, mask, seed):
    torch.manual_seed(seed)
    den.zero_grad(set_to_none=True)
    loss, _ = den(SimpleNamespace(obs=obs, act=act, mask_padding=mask))
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), torch.cat([p.grad.detach().flatten() for p in den.inner_model.parameters()])


def _train_denoiser(inner, dev, seed=3):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.synthetic import randomize_module_
    from oracle import torch_oracle as O

    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths),
                                                   inner.num_actions), 0.5, 0.3))
    randomize_module_(den.inner_model, seed)
    den = den.to(dev).train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    return den


def test_cond2048_uint8_batch_matches_fp32_twin():
    """Denoiser.forward at CC = 2048, two autoregressive steps, on a uint8 batch and on its fp32 decoding: the packed inputs are
    bit-identical (tests/test_gpu_uint8_frames.py), so loss and gradients differ only by the order of atomic additions."""
    from diamond_b200 import frames as F
    from oracle import torch_oracle as O

    dev = _dev()
    inner = O.InnerCfg(cond_channels=2048, depths=[1, 1, 1, 1], channels=[64, 128, 128, 128])
    den = _train_denoiser(inner, dev)
    b, t = 8, inner.num_steps_conditioning + 2
    rng = np.random.default_rng(17)
    levels = torch.from_numpy(rng.integers(0, 256, size=(b, t, inner.img_channels, 64, 64), dtype=np.uint8)).to(dev)
    act = torch.from_numpy(rng.integers(0, inner.num_actions, size=(b, t)).astype(np.int64)).to(dev)
    mask = torch.ones(b, t, dtype=torch.bool, device=dev)
    mask[0, :2] = False
    mask[1, t - 1:] = False
    twin = F.decode(levels, F.kinds_from_mask(mask, (b, t), dev))
    lf, gf = _den_step(den, twin, act, mask, 5)
    lf2, gf2 = _den_step(den, twin, act, mask, 5)
    lu, gu = _den_step(den, levels, act, mask, 5)
    within, cross = _rel(gf2, gf), _rel(gu, gf)
    print(f"CC=2048 uint8 vs fp32: loss {float(lu):.7f} vs {float(lf):.7f}; whole gradient {cross:.2e} (fp32 run-to-run {within:.2e})")
    assert torch.isfinite(gu).all()
    assert abs(float(lu) - float(lf)) <= 1e-6 * abs(float(lf))
    assert cross <= max(2 * within, 1e-5), (cross, within)


# a net whose dcond partials the backward temporary cannot hold: one 64-channel level at 8 x 8 (tA = B x 64 x 64 floats holds 2
# partials of B x 2048) with 3456 FiLM rows (13 splits), trained at batch 256
OWN_PARTIALS = dict(inner=dict(cond_channels=2048, depths=[4], channels=[64], attn_depths=[0]), h=8, w=8, b=256)


def _dcond_plan(inner, b, h, w, dev):
    """(splits, floats of the partials' own buffer, floats of the backward temporary) of the real training plan."""
    import ctypes

    from diamond_b200 import _lib
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig

    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths),
                                                   inner.num_actions), 0.5, 0.3)).to(dev)
    splits, own, tmp = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_longlong()
    lib = _lib.lib()
    _lib.check(lib.dmd_denoiser_train_dcond_plan(den.inner_model.native(), b, h, w, ctypes.byref(splits), ctypes.byref(own),
                                                 ctypes.byref(tmp)))
    return splits.value, own.value, tmp.value


def _want_splits(inner):
    from oracle import torch_oracle as O

    rows = sum(v[0] for k, v in O.inner_model_shapes(inner) if k.endswith(".linear.weight"))
    return min(32, rows // 256)


@pytest.mark.parametrize("label,inner,b,h,w", [
    ("default-b256", dict(), 256, 64, 64),
    ("wide-b32", dict(depths=[1, 1, 1, 1], channels=[64, 128, 128, 128]), 32, 64, 64),
    ("1level-8x8-c32", dict(cond_channels=256, depths=[4], channels=[32], attn_depths=[0]), 5, 8, 8),
    ("1level-8x8-c64", dict(cond_channels=256, depths=[4], channels=[64], attn_depths=[0]), 256, 8, 8),
    ("2level-16x16", dict(cond_channels=224, depths=[2, 2], channels=[32, 64], attn_depths=[0, 0]), 3, 16, 16),
])
def test_dcond_plan_at_cond_256_or_less_is_capped_by_the_temporary(label, inner, b, h, w):
    """Nets that trained before wider conditioning existed keep their dcond plan: the partials live in the backward temporary,
    and the split count is min(rows / 256 capped at 32, what the temporary holds), never below 8 of them."""
    from oracle import torch_oracle as O

    dev = _dev()
    inner = O.InnerCfg(**inner)
    splits, own, tmp = _dcond_plan(inner, b, h, w, dev)
    want, fit = _want_splits(inner), tmp // (b * inner.cond_channels)
    print(f"{label}: {splits} splits (rows / 256: {want}, the temporary holds {fit}), own buffer {own} floats")
    assert own == 0 and fit >= 8
    assert splits == min(want, fit)


def test_dcond_partials_past_the_temporary_get_their_own_buffer():
    from oracle import torch_oracle as O

    dev = _dev()
    c = OWN_PARTIALS
    inner = O.InnerCfg(**c["inner"])
    splits, own, tmp = _dcond_plan(inner, c["b"], c["h"], c["w"], dev)
    want = _want_splits(inner)
    print(f"own partials: {splits} splits of rows / 256 = {want}; own buffer {own} floats, temporary {tmp} floats")
    assert tmp // (c["b"] * 2048) < 8 and splits == want >= 8
    assert own == splits * c["b"] * 2048 and own > tmp
    # the default net at 64 x 64 keeps its partials in the temporary at every width
    for cc in (512, 2048):
        s2, own2, _ = _dcond_plan(O.InnerCfg(cond_channels=cc), 256, 64, 64, dev)
        assert (s2, own2) == (28, 0), (cc, s2, own2)


def test_cond2048_batch256_own_partials_step_against_float64():
    """The B = 256 step of OWN_PARTIALS, whose dcond = dfilm Wf partials have their own buffer (the test above).  dcond reaches
    the parameters only through cond_proj.2 (dW2 = dcond^T h), cond_proj.0 and act_emb; those and the FiLM gradients are checked
    against float64 autograd, as is the whole gradient, with the caps of tests/test_gpu_training_configs.py."""
    from oracle import torch_oracle as O
    from oracle import training_configs as TC

    dev = _dev()
    T = _load("test_gpu_training_configs")
    c = dict(OWN_PARTIALS, inner=O.InnerCfg(**OWN_PARTIALS["inner"]), seq=1, mask_off=[(3, 4), (200, 4)], wseed=697, dseed=698)
    loss, grads = T._native_denoiser(c, dev)
    T._threads()
    obs, act, mask, draws = TC.denoiser_inputs(c)
    sd = T._denoiser_sd(c)
    ref_loss, ref = O.denoiser_loss_grads_chunked(obs.double(), act, mask, [tuple(t.double() for t in d) for d in draws], sd,
                                                  O.DenoiserCfg(inner=c["inner"]), O.SigmaDistCfg(), 64)
    whole = T._rel_whole(grads, ref)
    cond_keys = [k for k in ref if k.startswith(("cond_proj", "act_emb"))]
    film_keys = [k for k in ref if k.endswith(".linear.weight") or k.endswith(".linear.bias")]
    e_cond = {k: _rel(grads[k], ref[k]) for k in cond_keys}
    e_film = max(_rel(grads[k], ref[k]) for k in film_keys)
    print(f"B=256 CC=2048 own partials: loss {loss:.6f} vs {ref_loss:.6f}; whole gradient {whole:.3e}; cond path {e_cond}; "
          f"worst FiLM {e_film:.3e}")
    assert abs(loss - ref_loss) <= 2e-3 * abs(ref_loss)
    assert whole < T.WHOLE_CAP, whole
    assert max(e_cond.values()) < T.PER_TENSOR_CAP and e_film < T.PER_TENSOR_CAP, (e_cond, e_film)


def _native_denoiser_uint8(c, dev):
    """tests/test_gpu_training_configs.py's native step on the case's frames as uint8 levels (every frame valid, so each level
    decodes to the float frame the oracle reads)."""
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from oracle import torch_oracle as O
    from oracle import training_configs as TC

    inner = c["inner"]
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths),
                                                   inner.num_actions), 0.5, 0.3))
    den.inner_model.load_state_dict(O.seeded_state_dict(O.inner_model_shapes(inner), c["wseed"]))
    den = den.to(dev).train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    obs, act, mask, draws = TC.denoiser_inputs(c)
    assert bool(mask.all())
    levels = ((obs + 1) / 2 * 255).round().to(torch.uint8)
    assert torch.equal(levels.float().div(255).mul(2).sub(1), obs)
    q = [t.to(dev) for d in draws for t in d]
    o1, o2 = torch.randn, torch.randn_like
    torch.randn = torch.randn_like = lambda *a, **k: q.pop(0).clone()
    try:
        loss, _ = den(SimpleNamespace(obs=levels.to(dev), act=act.to(dev), mask_padding=mask.to(dev)))
    finally:
        torch.randn, torch.randn_like = o1, o2
    assert not q, "Denoiser.forward consumed a different number of random draws"
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {k: p.grad.detach().cpu() for k, p in den.inner_model.named_parameters()}


def test_cond2048_uint8_batch_training_matches_float64_autograd(monkeypatch):
    """The [64, 128, 128, 128] net of the uint8 twin test above, CC = 2048, two autoregressive steps, trained on a uint8 batch and
    checked against float64 autograd with the fp16-emulation bounds of tests/test_gpu_training_configs.py."""
    import oracle.training_configs as TC
    from oracle import torch_oracle as O

    T = _load("test_gpu_training_configs")
    dev = _dev()
    c = dict(inner=O.InnerCfg(cond_channels=2048, depths=[1, 1, 1, 1], channels=[64, 128, 128, 128]), h=64, w=64, b=2, seq=2,
             mask_off=[], wseed=699, dseed=700)
    monkeypatch.setitem(TC.DENOISER_CASES, "C2u8", c)
    monkeypatch.setattr(T, "_native", lambda name, d: _native_denoiser_uint8(TC.DENOISER_CASES[name], d))
    T._check_case("C2u8", dev)


# ------------------------------------------------------------------------------------------------ accumulate / poisoned / views
def _patch_cond_nets(monkeypatch, GA):
    from oracle import torch_oracle as O

    inner, rew = GA._inner_cfg, GA._rew_end_cfg
    nets = {"cond2048": (O.InnerCfg(cond_channels=2048, depths=[1, 1, 1, 1], channels=[64, 128, 128, 128]), 2, 64),
            "own_partials": (O.InnerCfg(**OWN_PARTIALS["inner"]), OWN_PARTIALS["b"], OWN_PARTIALS["h"])}
    monkeypatch.setattr(GA, "_inner_cfg", lambda name: nets[name] if name in nets else inner(name))
    monkeypatch.setattr(GA, "_rew_end_cfg", lambda name: O.RewEndCfg(cond_channels=2048) if name == "cond2048" else rew(name))


@pytest.mark.parametrize("model", ["denoiser", "rew_end"])
def test_cond2048_accumulate_entry_point_adds_the_plain_result(model, monkeypatch):
    GA = _load("test_gpu_grad_accumulation")
    _patch_cond_nets(monkeypatch, GA)
    GA.test_accumulate_entry_point_adds_the_plain_result(model, "cond2048")


@pytest.mark.parametrize("byte", [0xFF, 0x5A], ids=lambda b: f"0x{b:02X}")
@pytest.mark.parametrize("model,net", [("denoiser", "cond2048"), ("rew_end", "cond2048"), ("denoiser", "own_partials")])
def test_cond2048_on_poisoned_workspace_and_outputs(model, net, byte, monkeypatch):
    """Workspace, outputs and g_*_in poisoned before forward_train + backward_accumulate at CC = 2048 (the split-K partials of
    dcond, in the backward temporary or, for own_partials, in their own buffer, and the FiLM and cond-MLP scratch) give what
    clean memory gives."""
    from test_gpu_poisoned_buffers import poison_

    GA = _load("test_gpu_grad_accumulation")
    _patch_cond_nets(monkeypatch, GA)
    dev = _dev()
    c = GA._calls(model, net, dev)

    def run(p):
        acc = torch.ones(c.total, device=dev)
        if p is not None:
            poison_(c.ws, p)
            for t in c.outs if model == "rew_end" else [c.out]:
                poison_(t, p)
            for t in getattr(c, "g_in", []):
                poison_(t, p)
        c.forward()
        c.L.check(c.backward(True, acc.data_ptr(), c.total))
        torch.cuda.synchronize()
        return GA._split(acc, c.layout) + [x.clone() for x in getattr(c, "g_in", [])]

    ref, again = run(None), run(None)
    GA._check(f"{model} {net} poisoned 0x{byte:02X}", run(byte), ref, again)


def test_cond2048_autoregressive_steps_share_one_flat_buffer():
    """Two autoregressive steps (two native nodes) under one loss.backward(): one flat buffer, every .grad a view of it, equal to
    torch.autograd.grad of the same loss."""
    from oracle import torch_oracle as O

    GA = _load("test_gpu_grad_accumulation")
    dev = _dev()
    inner = O.InnerCfg(cond_channels=2048, depths=[1, 1, 1], channels=[32, 64, 128], attn_depths=[0, 0, 0])
    den = _train_denoiser(inner, dev)
    params = list(den.parameters())
    batch = GA._den_batch(inner, 3, 32, 2, 41, dev)
    ref = torch.autograd.grad(GA._den_loss(den, batch, 7), params)
    again = torch.autograd.grad(GA._den_loss(den, batch, 7), params)
    GA._den_loss(den, batch, 7).backward()
    torch.cuda.synchronize()
    GA._check("CC=2048 two autoregressive steps", [p.grad for p in params], ref, again)
    assert GA._aliases_last_flat_grad(den.inner_model)
    flat = den.inner_model.last_flat_grad
    film = den.inner_model.unet.d_blocks[0].resblocks[0].norm1.linear.weight
    assert film.shape[1] == 2048 and film.grad.data_ptr() >= flat.data_ptr()
    assert not math.isnan(float(flat.sum()))
