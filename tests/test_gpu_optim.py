"""GPU: the native optimizer (diamond_b200/optim.py on csrc/optim_kernels.cuh) against torch's clip_grad_norm_ /
torch.optim.AdamW(foreach=False) and the float64 restatement (oracle/optim_reference.py), on the gradient layouts of the three
trained models: the flat buffer the native backward fills (numels that are not multiples of 4, 1-element tensors), gradients
outside it, and None gradients."""
import io

import pytest
import torch

from diamond_b200 import _lib, optim
from oracle import optim_reference as OR

pytestmark = pytest.mark.gpu

LR, WD, EPS = 1e-4, 1e-2, 1e-8


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _model(kind, dev, seed=2024):
    """(module, native module whose flat gradient layout the parameters use) at each model's default config."""
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import randomize_module_

    if kind == "denoiser":
        m = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [2, 2, 2, 2], [64] * 4, [0] * 4, 4), 0.5, 0.3))
        randomize_module_(m.inner_model, seed)
        m = m.to(dev)
        return m, m.inner_model
    if kind == "actor_critic":
        m = ActorCritic(ActorCriticConfig(512, 3, 64, [32, 32, 64, 64], [1, 1, 1, 1], 4))
    else:
        m = RewEndModel(RewEndModelConfig(512, 3, 64, 128, [2, 2, 2, 2], [32] * 4, [0] * 4, 4))
    randomize_module_(m, seed)
    m = m.to(dev)
    return m, m


def _flat_grads(native, params, seed, none=(), separate=()):
    """Gradients as the native backward leaves them: views of one flat buffer at the model's layout, each tensor at its own
    scale; indices in `none` get no gradient, those in `separate` a tensor of their own (what gradient accumulation leaves)."""
    offs, nums, total = native._grad_views_layout()
    gen = torch.Generator(device=params[0].device).manual_seed(seed)
    flat = torch.randn(total, generator=gen, device=params[0].device)
    for i, (o, n) in enumerate(zip(offs, nums)):
        flat[o:o + n] *= 10.0 ** ((i % 7) - 4)
    for i, (p, o, n) in enumerate(zip(params, offs, nums)):
        g = flat[o:o + n].view_as(p)
        p.grad = None if i in none else (g.clone() if i in separate else g)
    return flat


def _f64_norm(grads):
    return float(torch.sqrt(sum((g.double() ** 2).sum() for g in grads)))


def _ulps(a, b, floor=0.0):
    """Largest elementwise distance in units of the fp32 spacing at max(|b|, floor) (at least the smallest normal's).  For
    parameters the floor is the learning rate: where an update cancels a parameter down to near zero, the distance is
    measured in ulps of the update, not of the small remainder."""
    a, b = a.detach().float().reshape(-1), b.detach().float().reshape(-1)
    mag = torch.maximum(b.abs(), torch.full_like(b, max(floor, torch.finfo(torch.float32).tiny)))
    spacing = torch.nextafter(mag, torch.full_like(mag, float("inf"))) - mag
    return float(((a.double() - b.double()).abs() / spacing.double()).max()) if a.numel() else 0.0


@pytest.mark.parametrize("kind", ["denoiser", "actor_critic", "rew_end"])
def test_clip_norm_matches_float64_on_model_layouts(kind):
    dev = _dev()
    model, native = _model(kind, dev)
    params = list(native.parameters())
    assert kind == "rew_end" or any(p.numel() % 4 for p in params)   # the reward/termination model has none
    _flat_grads(native, params, 7, none={3}, separate={0, 5, len(params) - 1})
    grads = [p.grad for p in params if p.grad is not None]
    before = [g.clone() for g in grads]
    want = _f64_norm(grads)
    max_norm = 0.5 * want
    lib = _lib.lib()
    lib.dmd_launch_count(1)
    total = optim.clip_grad_norm_(params, max_norm)
    launches = lib.dmd_launch_count(1)
    torch.cuda.synchronize()
    assert total.device == dev and total.dtype == torch.float32 and total.dim() == 0
    assert launches == 3
    assert abs(float(total) - want) <= 1e-6 * want, (float(total), want)
    coef = max_norm / (want + 1e-6)
    worst = max(float((g.double() - b.double() * coef).norm() / (b.double() * coef).norm()) for g, b in zip(grads, before))
    print(f"{kind}: {len(grads)} gradients, norm rel err {abs(float(total) - want) / want:.2e}, worst clipped tensor {worst:.2e}")
    assert worst < 1e-6
    # torch's own clip on the same gradients: the coefficient agrees to fp32 rounding
    ref = [b.clone() for b in before]
    ref_total = torch.nn.utils.clip_grad_norm_([_with_grad(r) for r in ref], max_norm)
    assert abs(float(ref_total) - float(total)) <= 1e-5 * want
    # a second run on the same inputs is bit-identical
    for g, b in zip(grads, before):
        g.copy_(b)
    again = optim.clip_grad_norm_(params, max_norm)
    assert torch.equal(again, total)


def _with_grad(g):
    p = torch.nn.Parameter(torch.zeros_like(g))
    p.grad = g
    return p


def test_clip_repeat_runs_are_bit_identical_and_inactive_clip_leaves_grads():
    dev = _dev()
    model, native = _model("denoiser", dev)
    params = list(native.parameters())
    _flat_grads(native, params, 11)
    before = [p.grad.clone() for p in params]
    totals = []
    for _ in range(3):
        for p, b in zip(params, before):
            p.grad.copy_(b)
        totals.append(optim.clip_grad_norm_(params, 1e30))
    assert all(torch.equal(t, totals[0]) for t in totals)
    assert all(torch.equal(p.grad, b) for p, b in zip(params, before))


@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_clip_propagates_inf_and_nan_as_torch_does(bad):
    dev = _dev()
    gen = torch.Generator(device=dev).manual_seed(3)
    gs = [torch.randn(n, generator=gen, device=dev) for n in (1, 7, 40000, 13)]
    gs[2][12345] = bad
    ours = [_with_grad(g.clone()) for g in gs]
    theirs = [_with_grad(g.clone()) for g in gs]
    t_ours = optim.clip_grad_norm_(ours, 1.0)
    t_theirs = torch.nn.utils.clip_grad_norm_(theirs, 1.0)
    torch.testing.assert_close(t_ours, t_theirs, equal_nan=True, rtol=0, atol=0)
    for a, b in zip(ours, theirs):
        torch.testing.assert_close(a.grad, b.grad, equal_nan=True, rtol=0, atol=0)
    with pytest.raises(RuntimeError, match="non-finite"):
        optim.clip_grad_norm_([_with_grad(g.clone()) for g in gs], 1.0, error_if_nonfinite=True)


def _twin(params, dev):
    return [torch.nn.Parameter(p.detach().clone()) for p in params]


@pytest.mark.parametrize("kind", ["denoiser", "actor_critic", "rew_end"])
def test_adamw_matches_torch(kind):
    """3 steps with the configure_opt groups (lr 1e-4, wd 1e-2, eps 1e-8): p, m, v within a few ulps of
    torch.optim.AdamW(foreach=False) on identical fp32 inputs; one 1-element and one None-gradient tensor included.  The
    moments come out bit-identical; the parameters differ from torch's in the last bits where the rounding of the update's
    last operations differs (at most 6 ulps of max(|p|, lr) after 3 steps on an H100)."""
    dev = _dev()
    model, native = _model(kind, dev)
    groups = OR.configure_opt_groups(model, WD)
    order = [p for g in groups for p in g["params"]]
    twin = _twin(order, dev)
    twin_groups, k = [], 0
    for g in groups:
        twin_groups.append({"params": twin[k:k + len(g["params"])], "weight_decay": g["weight_decay"]})
        k += len(g["params"])
    ours = optim.AdamW(groups, lr=LR, eps=EPS)
    ref = torch.optim.AdamW(twin_groups, lr=LR, eps=EPS, foreach=False)
    params = list(native.parameters())
    skip = {i for i, p in enumerate(order) if p is params[2]}
    for step in range(3):
        _flat_grads(native, params, 100 + step, none={2})
        for p, t in zip(order, twin):
            t.grad = None if p.grad is None else p.grad.clone()
        ours.step()
        ref.step()
    torch.cuda.synchronize()
    worst = {"p": 0.0, "m": 0.0, "v": 0.0}
    for i, (p, t) in enumerate(zip(order, twin)):
        if i in skip:
            assert p not in ours.state or not ours.state[p]
            continue
        worst["p"] = max(worst["p"], _ulps(p, t, LR))
        worst["m"] = max(worst["m"], _ulps(ours.state[p]["exp_avg"], ref.state[t]["exp_avg"]))
        worst["v"] = max(worst["v"], _ulps(ours.state[p]["exp_avg_sq"], ref.state[t]["exp_avg_sq"]))
        assert float(ours.state[p]["step"]) == float(ref.state[t]["step"]) == 3.0
    print(f"{kind}: worst ulps vs torch foreach=False {worst}")
    assert worst["p"] <= 8 and worst["m"] <= 1 and worst["v"] <= 1, worst   # H100: 5-6 / 0 / 0


def test_adamw_cumulative_update_matches_float64():
    """Against the float64 restatement, on the configure_opt groups of the actor-critic and with a clip active: relative L2 of
    the cumulative update within 1e-6.  lr 1e-2 here: at lr 1e-4 the fp32 storage of the parameters alone (half an ulp of
    |p| per step) is ~1e-5 of a 3-step update, for torch's optimizer as for this one."""
    dev = _dev()
    model, native = _model("actor_critic", dev)
    groups = OR.configure_opt_groups(model, WD)
    order = [p for g in groups for p in g["params"]]
    wds = [g["weight_decay"] for g in groups for _ in g["params"]]
    start = [p.detach().clone() for p in order]
    ours = optim.AdamW(groups, lr=1e-2, eps=EPS)
    params = list(native.parameters())
    grads_per_step = []
    for step in range(3):
        _flat_grads(native, params, 200 + step)
        grads_per_step.append([p.grad.detach().clone() for p in order])
        optim.clip_grad_norm_(order, 0.5 * _f64_norm([p.grad for p in order]))
        ours.step()
    want, _, _ = OR.train_steps(start, [OR.clip_grad_norm(g, 0.5 * _f64_norm(g))[0] for g in grads_per_step], wds, None, 1e-2)
    num = sum(float(((p.detach().double() - w) ** 2).sum()) for p, w in zip(order, want))
    den = sum(float(((w - s.double()) ** 2).sum()) for w, s in zip(want, start))
    print(f"cumulative update rel L2 vs float64: {(num / den) ** 0.5:.2e}")
    assert (num / den) ** 0.5 < 1e-6


def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=True)


@pytest.mark.parametrize("direction", ["native_to_torch", "torch_to_native"])
def test_state_dict_round_trip_with_torch(direction):
    dev = _dev()
    model, native = _model("rew_end", dev)
    groups = OR.configure_opt_groups(model, WD)
    order = [p for g in groups for p in g["params"]]
    params = list(native.parameters())

    def make(cls, ps, **kw):
        out, k = [], 0
        for g in groups:
            out.append({"params": ps[k:k + len(g["params"])], "weight_decay": g["weight_decay"]})
            k += len(g["params"])
        return cls(out, lr=LR, eps=EPS, **kw)

    first_cls, first_kw = (optim.AdamW, {}) if direction == "native_to_torch" else (torch.optim.AdamW, {"foreach": False})
    second_cls, second_kw = (torch.optim.AdamW, {"foreach": False}) if direction == "native_to_torch" else (optim.AdamW, {})
    first = make(first_cls, order, **first_kw)
    for step in range(2):
        _flat_grads(native, params, 300 + step)
        first.step()
    # continue twice: with the first optimizer, and with a second one of the other kind loaded from its checkpoint
    twin = _twin(order, dev)
    second = make(second_cls, twin, **second_kw)
    second.load_state_dict(_roundtrip(first.state_dict()))
    assert second.state_dict()["param_groups"][0]["weight_decay"] == WD
    if isinstance(second, optim.AdamW):
        m_flat = second._flat[0]
        lo, hi = m_flat.data_ptr(), m_flat.data_ptr() + 4 * m_flat.numel()
        assert all(lo <= second.state[t]["exp_avg"].data_ptr() < hi for t in twin)
    for step in range(2):
        _flat_grads(native, params, 400 + step)
        for p, t in zip(order, twin):
            t.grad = p.grad.clone()
        first.step()
        second.step()
    worst = max(_ulps(t, p, LR) for p, t in zip(order, twin))
    worst_m = max(_ulps(second.state[t]["exp_avg_sq"], first.state[p]["exp_avg_sq"]) for p, t in zip(order, twin))
    print(f"{direction}: worst ulps p {worst}, v {worst_m}")
    assert worst <= 8 and worst_m <= 1
    assert all(float(second.state[t]["step"]) == 4.0 for t in twin)


def _denoiser_forward(den, dev):
    from diamond_b200.synthetic import frame_stacks

    obs, act, x0 = frame_stacks(2, 4, 3, 64, 64, 4, 5)
    sigma = torch.tensor([0.7], device=dev)
    with torch.no_grad():
        out, _ = den._native_forward(x0.to(dev), sigma, obs.reshape(2, -1, 64, 64).to(dev), act.to(dev), True, False)
    torch.cuda.synchronize()
    return out.clone()


def test_native_step_repacks_the_denoisers_weights():
    """A denoiser forward after a native step equals one after a torch step on the same gradients; without the version bump
    the native model would still run the packed fp16 weights of before the step."""
    dev = _dev()
    den_a, native_a = _model("denoiser", dev)
    den_b, native_b = _model("denoiser", dev)
    before = _denoiser_forward(den_a, dev)
    pa, pb = list(native_a.parameters()), list(native_b.parameters())
    _flat_grads(native_a, pa, 500)
    for p, q in zip(pa, pb):
        q.grad = p.grad.clone()
    optim.AdamW(OR.configure_opt_groups(den_a, WD), lr=1e-3, eps=EPS).step()
    torch.optim.AdamW(OR.configure_opt_groups(den_b, WD), lr=1e-3, eps=EPS, foreach=False).step()
    after_a, after_b = _denoiser_forward(den_a, dev), _denoiser_forward(den_b, dev)
    moved = float((after_b - before).norm() / before.norm())
    diff = float((after_a - after_b).norm() / after_b.norm())
    print(f"re-pack: step moved the output by {moved:.2e}; native vs torch step {diff:.2e}")
    assert moved > 1e-3
    assert diff < 0.01 * moved


def test_gradient_accumulation_then_step():
    """Two Denoiser.forward + backward before one clip + step: the gradients stop aliasing the flat backward buffer, the table
    is rebuilt, and the step matches torch's on the same gradients; then a fresh single backward (aliasing again)."""
    from diamond_b200.models.diffusion import SigmaDistributionConfig
    from diamond_b200.synthetic import frame_stacks

    dev = _dev()
    den, native = _model("denoiser", dev)
    den.train().setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))
    obs, act, _ = frame_stacks(4, 5, 3, 64, 64, 4, 77)

    class B_:
        pass

    batch = B_()
    batch.obs, batch.act, batch.mask_padding = obs.to(dev), act.to(dev), torch.ones(4, 5, dtype=torch.bool, device=dev)
    params = list(native.parameters())
    twin = _twin(params, dev)
    ours = optim.AdamW(OR.configure_opt_groups(den, WD), lr=LR, eps=EPS)
    names = {id(p): i for i, p in enumerate(params)}
    twin_groups = [{"params": [twin[names[id(p)]] for p in g["params"]], "weight_decay": g["weight_decay"]}
                   for g in OR.configure_opt_groups(den, WD)]
    ref = torch.optim.AdamW(twin_groups, lr=LR, eps=EPS, foreach=False)
    for backwards in (2, 1):
        ours.zero_grad(set_to_none=True)
        for k in range(backwards):
            torch.manual_seed(k)
            den(batch)[0].backward()
        flat = native.last_flat_grad
        lo, hi = flat.data_ptr(), flat.data_ptr() + 4 * flat.numel()
        aliased = all(lo <= p.grad.data_ptr() < hi for p in params)
        assert aliased == (backwards == 1)
        for p, t in zip(params, twin):
            t.grad = p.grad.clone()
        n_ours = optim.clip_grad_norm_(params, 1.0)
        n_ref = torch.nn.utils.clip_grad_norm_(twin, 1.0)
        assert abs(float(n_ours) - float(n_ref)) <= 1e-5 * float(n_ref)
        ours.step()
        ref.step()
        worst = max(_ulps(p, t, LR) for p, t in zip(params, twin))
        print(f"{backwards} backward(s): norm {float(n_ours):.4g}, worst ulps vs torch {worst}")
        assert worst <= 8


def test_launches_per_step_do_not_depend_on_the_tensor_count():
    """clip + step is 3 + 1 launches for 10 tensors and for the denoiser's 235."""
    dev = _dev()
    _, native = _model("denoiser", dev)
    big = list(native.parameters())
    small = [_with_grad(torch.randn(n, device=dev)) for n in (1, 3, 4, 5, 17, 64, 1000, 4097, 16385, 70000)]
    _flat_grads(native, big, 600)
    lib = _lib.lib()
    counts = []
    for ps in (small, big):
        opt = optim.AdamW(ps, lr=LR, weight_decay=WD, eps=EPS)
        for _ in range(2):   # the second step reuses the table
            lib.dmd_launch_count(1)
            optim.clip_grad_norm_(ps, 1.0)
            opt.step()
            counts.append(lib.dmd_launch_count(1))
    assert len(big) == 235
    assert counts == [4, 4, 4, 4], counts
