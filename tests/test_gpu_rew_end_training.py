"""GPU: RewEndModel training (rew_end_model.py:57-90) on the native path -- dmd_rew_end_forward_train / dmd_rew_end_backward
behind one autograd node -- against the reference golden (tests/golden/rew_end_training.npz), and at the trainer's shape
(32 segments x seq_length 19, trainer.yaml:108,113) against the fp32 oracle accumulated over groups of segments."""
import time

import numpy as np
import pytest
import torch

from oracle import torch_oracle as O
from oracle import rew_end_training as RT

pytestmark = pytest.mark.gpu

PER_TENSOR_CAP = 5e-3   # as tests/test_gpu_training.py: no tensor's relative L2 error may exceed this


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


class _Batch:
    def __init__(self, obs, act, rew, end, mask, info):
        self.obs, self.act, self.rew, self.end, self.mask_padding, self.info = obs, act, rew, end, mask, info
        self.trunc = torch.zeros_like(end)


def _model(cfg, sd, dev):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig

    m = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                      list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
    m.load_state_dict(sd)
    return m.to(dev).train()


def _batch(obs, act, rew, end, mask, final_obs, dev):
    info = [{"final_observation": final_obs[i].to(dev)} if i in final_obs else {} for i in range(obs.size(0))]
    return _Batch(obs.to(dev).clone(), act.to(dev), rew.to(dev), end.to(dev), mask.to(dev), info)


def _native_step(model, batch):
    """RewEndModel.forward + backward; also returns the logits the autograd node produced."""
    seen = {}
    inner = model.predict_rew_end

    def tap(*a, **k):
        out = inner(*a, **k)
        seen["logits"] = (out[0].detach(), out[1].detach())
        return out
    model.predict_rew_end = tap
    try:
        loss, metrics = model(batch)
    finally:
        del model.predict_rew_end
    model.zero_grad(set_to_none=True)
    loss.backward()
    torch.cuda.synchronize()
    return loss, metrics, seen["logits"]


def _seeded_batch(b, T, seed):
    """b segments of T frames at the default config: every fourth segment dies at a random step (its later frames padding),
    every fifth runs past its episode's end (padding from a random step on), rewards of every sign."""
    cfg = O.RewEndCfg()
    rng = np.random.default_rng(seed)
    obs_u8 = rng.integers(0, 256, size=(b, T, cfg.img_channels, cfg.img_size, cfg.img_size), dtype=np.uint8)
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, T)).astype(np.int64))
    rew = torch.from_numpy(rng.choice([-2.0, -1.0, 0.0, 0.0, 0.0, 1.0, 3.0], size=(b, T)).astype(np.float32))
    end = torch.zeros(b, T, dtype=torch.long)
    mask = torch.ones(b, T, dtype=torch.bool)
    final_obs = {}
    for i in range(b):
        if i % 4 == 1:
            t0 = int(rng.integers(0, T - 1))
            end[i, t0] = 1
            final_obs[i] = RT.frames(rng.integers(0, 256, size=obs_u8.shape[2:], dtype=np.uint8))
            pad = t0 + 1
        elif i % 5 == 2:
            pad = int(rng.integers(2, T))
        else:
            continue
        mask[i, pad:] = False
        obs_u8[i, pad:] = 127
        rew[i, pad:] = 0
        act[i, pad:] = 0
    return RT.frames(obs_u8), act, rew, end, mask, final_obs


# native logits lie within this many ensemble spreads of the fp16-operand emulation: 1.5 x (5.75e-4, 4.13e-4) is tighter than the
# old 1e-3 against the reference, and still admits a regrouping of the GroupNorm partial sums
SPREAD_MULTIPLE = 1.5


def test_rew_end_training_step_matches_reference():
    """The logits are bounded by what the native operand rounding produces (oracle/fp16_emulation.py, derived on the CPU in
    tests/test_oracle_rew_end_training.py::test_rew_end_logits_bound_from_fp16_emulation): against the reference's fp32 logits
    within 1.5 x the worst distance of the fp16-operand emulation ensemble (1.66e-3 rew, 1.19e-3 end), and against the
    unperturbed emulation within SPREAD_MULTIPLE x the ensemble's spread (5.75e-4 rew, 4.13e-4 end).  Measured on an H100
    80GB HBM3 (700 W power limit): 9.73e-4 / 6.44e-4 from the reference, 5.52e-4 / 3.38e-4 from the emulation; with the
    all-padding tail tile dropped from the conv schedule (a regrouping of the fp32 GroupNorm partial sums) 1.08e-3 / 6.95e-4
    and 5.92e-4 / 3.50e-4, inside both bounds."""
    from oracle import fp16_emulation as E

    dev = _dev()
    (obs, act, rew, end, mask, final_obs), g = RT.load_golden()
    cfg = O.RewEndCfg()
    model = _model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 778), dev)
    batch = _batch(obs, act, rew, end, mask, final_obs, dev)
    loss, metrics, (lr, le) = _native_step(model, batch)
    e_loss = abs(loss.item() - float(g["loss"])) / abs(float(g["loss"]))
    e_rew, e_end = _rel(lr, torch.from_numpy(g["logits_rew"])), _rel(le, torch.from_numpy(g["logits_end"]))
    torch.set_num_threads(16)
    bound, spread, emu = E.rew_end_logits_bounds()
    d_rew, d_end = _rel(lr, emu[0]), _rel(le, emu[1])
    print(f"rew_end golden: loss {loss.item():.6f} reference {float(g['loss']):.6f} (rel {e_loss:.2e}); logits rel {e_rew:.2e} {e_end:.2e} "
          f"(bound {bound['rew']:.2e} {bound['end']:.2e}); from the emulation {d_rew:.2e} {d_end:.2e} "
          f"(spread {spread['rew']:.2e} {spread['end']:.2e})")
    assert e_loss < 1e-3
    assert e_rew <= bound["rew"] and e_end <= bound["end"], (e_rew, e_end, bound)
    assert d_rew <= SPREAD_MULTIPLE * spread["rew"] and d_end <= SPREAD_MULTIPLE * spread["end"], (d_rew, d_end, spread)
    assert torch.equal(batch.obs.cpu(), RT.frames(g["obs_substituted_u8"]))
    named = [(k, p.grad.cpu()) for k, p in model.named_parameters()]
    keys, norms, _ = O.grad_summary(named)
    assert keys == [str(k) for k in g["grad_keys"]]
    ref_n = g["grad_norms"]
    tot = float(np.sqrt((ref_n ** 2).sum()))
    rel_n = np.abs(norms - ref_n) / (ref_n + 1e-30)
    print("worst tensor norms:", sorted(zip(rel_n.tolist(), keys), reverse=True)[:3])
    assert np.all(np.abs(norms - ref_n) <= 4e-3 * ref_n + 1e-4 * tot), float(np.max(rel_n))
    # the flat buffer is what the parameters' .grad are views of
    flat = model.last_flat_grad
    assert all(p.grad.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr() for p in model.parameters())


def test_rew_end_training_trainer_shape_matches_oracle():
    """32 segments x 19 frames = 18 transitions per segment, 576 encoder rows: the oracle's fp32 gradient is accumulated over
    groups of 8 segments on the host (RT.rew_end_loss_grads_chunked)."""
    dev = _dev()
    cfg = O.RewEndCfg()
    inputs = _seeded_batch(32, 19, 1900)
    model = _model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 779), dev)
    t0 = time.perf_counter()
    loss, _, _ = _native_step(model, _batch(*inputs, dev))
    t1 = time.perf_counter()
    torch.set_num_threads(16)
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 779)
    for v in sd.values():
        v.requires_grad_(True)
    ref_loss, ref = RT.rew_end_loss_grads_chunked(*inputs, sd, cfg, chunk=8)
    t2 = time.perf_counter()
    grads = {k: p.grad.detach().cpu() for k, p in model.named_parameters()}
    num = den = 0.0
    rows = []
    for k in ref:
        d = grads[k].double() - ref[k].double()
        num += float(d.pow(2).sum()); den += float(ref[k].double().pow(2).sum())
        rows.append((float(d.norm() / ref[k].double().norm().clamp_min(1e-30)), k))
    whole = (num / den) ** 0.5
    e_loss = abs(loss.item() - ref_loss) / abs(ref_loss)
    worst = sorted(rows, reverse=True)[:5]
    print(f"rew_end 32x19: loss rel {e_loss:.2e}, whole-gradient rel {whole:.3e}, worst {worst}; native {t1 - t0:.2f} s, oracle {t2 - t1:.1f} s")
    assert e_loss < 1e-3
    assert whole < 1e-3, whole
    for e, k in rows:
        assert e < PER_TENSOR_CAP, (k, e)


def test_rew_end_two_optimizer_steps_match_oracle():
    """clip_grad_norm_(100) + AdamW (trainer.yaml's rew_end optimizer: lr 1e-4, weight decay 1e-2, eps 1e-8) twice: the weights
    re-pack after each step and the loss of the step after them matches the oracle's."""
    dev = _dev()
    (obs, act, rew, end, mask, final_obs), _ = RT.load_golden()
    cfg = O.RewEndCfg()
    model = _model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 778), dev)
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 778)
    for v in sd.values():
        v.requires_grad_(True)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=1e-2, eps=1e-8)
    names = [k for k, _ in model.named_parameters()]
    opt_ref = torch.optim.AdamW([sd[k] for k in names], lr=1e-4, weight_decay=1e-2, eps=1e-8)
    losses = []
    for step in range(3):
        loss, _, _ = _native_step(model, _batch(obs, act, rew, end, mask, final_obs, dev))
        ref_loss = RT.rew_end_loss(obs, act, rew, end, mask, final_obs, sd, cfg)[0]
        losses.append((loss.item(), ref_loss.item()))
        if step == 2:
            break
        opt_ref.zero_grad()
        ref_loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 100.0)
        torch.nn.utils.clip_grad_norm_([sd[k] for k in names], 100.0)
        opt.step(); opt_ref.step()
    print("losses (native, oracle) per step:", losses)
    assert losses[2][0] != losses[0][0]
    for a, b in losses:
        assert abs(a - b) <= 1e-3 * abs(b), (a, b)


def test_rew_end_autograd_grad_and_carried_state():
    """torch.autograd.grad through predict_rew_end returns the flat buffer's values; the gradients wrt a carried (hx, cx)
    match float64 autograd of the oracle."""
    dev = _dev()
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 780)
    model = _model(cfg, sd, dev)
    b, t = 2, 3
    rng = np.random.default_rng(781)
    frames = RT.frames(rng.integers(0, 256, size=(b, t + 1, 3, 64, 64), dtype=np.uint8))
    act = torch.from_numpy(rng.integers(0, cfg.num_actions, size=(b, t)).astype(np.int64))
    hx = torch.from_numpy(rng.standard_normal((1, b, cfg.lstm_dim)).astype(np.float32)) * 0.3
    cx = torch.from_numpy(rng.standard_normal((1, b, cfg.lstm_dim)).astype(np.float32)) * 0.3
    w_rew, w_end = torch.randn(b, t, 3, generator=torch.Generator().manual_seed(7)), torch.randn(b, t, 2, generator=torch.Generator().manual_seed(8))
    w_h, w_c = (torch.randn(1, b, cfg.lstm_dim, generator=torch.Generator().manual_seed(s)) for s in (9, 10))

    def objective(lr, le, h, c, m):
        return (lr * m(w_rew)).sum() + (le * m(w_end)).sum() + (h * m(w_h)).sum() + (c * m(w_c)).sum()
    hx_d, cx_d = hx.to(dev).requires_grad_(True), cx.to(dev).requires_grad_(True)
    lr, le, (h, c) = model.predict_rew_end(frames[:, :-1].to(dev), act.to(dev), frames[:, 1:].to(dev), (hx_d, cx_d))
    params = list(model.parameters())
    gs = torch.autograd.grad(objective(lr, le, h, c, lambda x: x.to(dev)), [hx_d, cx_d] + params)
    flat = model.last_flat_grad
    offs, nums, _ = model._grad_views_layout()
    for gp, o, n in zip(gs[2:], offs, nums):
        assert torch.equal(gp.flatten(), flat[o:o + n])
    sd64 = {k: v.double() for k, v in sd.items()}
    hx64, cx64 = hx.double().requires_grad_(True), cx.double().requires_grad_(True)
    lr64, le64, (h64, c64) = O.predict_rew_end(frames[:, :-1].double(), act, frames[:, 1:].double(), sd64, cfg, (hx64, cx64))
    ghx, gcx = torch.autograd.grad(objective(lr64, le64, h64, c64, lambda x: x.double()), [hx64, cx64])
    e_h, e_c = _rel(gs[0], ghx), _rel(gs[1], gcx)
    print(f"carried state gradients vs float64: hx {e_h:.2e}, cx {e_c:.2e}")
    # the LSTM and head backward are fp32, but the gates they differentiate read the encoder's features, whose fp16-operand
    # forward carries the logits' 1e-3-level error (tests/test_gpu_rew_end.py bounds those logits by 2e-3)
    assert e_h < 2e-3 and e_c < 2e-3


def test_rew_end_inference_untouched_by_training():
    """predict_rew_end under no_grad after a training step on the same module (and its workspace pool) returns exactly what a
    fresh module returns."""
    dev = _dev()
    (obs, act, rew, end, mask, final_obs), _ = RT.load_golden()
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 778)
    trained, fresh = _model(cfg, sd, dev), _model(cfg, sd, dev)
    _native_step(trained, _batch(obs, act, rew, end, mask, final_obs, dev))
    args = (obs[:, :-1].to(dev), act[:, :-1].to(dev), obs[:, 1:].to(dev))
    with torch.no_grad():
        a, b_ = trained.predict_rew_end(*args), fresh.predict_rew_end(*args)
    for x, y in ((a[0], b_[0]), (a[1], b_[1]), (a[2][0], b_[2][0]), (a[2][1], b_[2][1])):
        assert torch.equal(x, y)


def test_rew_end_backward_rejections():
    from diamond_b200 import _lib

    dev = _dev()
    cfg = O.RewEndCfg()
    model = _model(cfg, O.seeded_state_dict(O.rew_end_shapes(cfg), 778), dev)
    lib, h = _lib.lib(), model._native()
    b, t = 2, 3
    offs, nums, total = model._grad_views_layout()
    flat = torch.empty(total, device=dev)
    g_rew, g_end = torch.zeros(b, t, 3, device=dev), torch.zeros(b, t, 2, device=dev)
    ws = torch.empty(lib.dmd_rew_end_train_workspace_bytes(h, b, t), dtype=torch.uint8, device=dev)
    st = _lib.current_stream()

    def backward(bb, tt, n=total):
        return lib.dmd_rew_end_backward(h, bb, tt, g_rew.data_ptr(), g_end.data_ptr(), None, None, flat.data_ptr(), n, None, None,
                                        ws.data_ptr(), st)
    assert backward(b, t) != 0 and "no matching dmd_rew_end_forward_train" in lib.dmd_last_error().decode()
    obs = torch.zeros(b, t, 3, 64, 64, device=dev)
    act = torch.zeros(b, t, dtype=torch.long, device=dev)
    outs = [torch.empty(b, t, 3, device=dev), torch.empty(b, t, 2, device=dev), torch.empty(b, 512, device=dev), torch.empty(b, 512, device=dev)]
    _lib.check(lib.dmd_rew_end_forward_train(h, b, t, obs.data_ptr(), obs.data_ptr(), act.data_ptr(), None, None,
                                             *[o.data_ptr() for o in outs], ws.data_ptr(), ws.numel(), st))
    assert backward(t, b) != 0 and "no matching dmd_rew_end_forward_train" in lib.dmd_last_error().decode()
    assert backward(b, t, total - 1) != 0 and "gradient buffer too small" in lib.dmd_last_error().decode()
    _lib.check(backward(b, t))
    torch.cuda.synchronize()
