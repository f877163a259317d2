"""GPU: native gradient accumulation of the denoiser and the reward / termination model -- dmd_denoiser_backward_accumulate /
dmd_rew_end_backward_accumulate at the C ABI, the nodes of one `loss.backward()` adding into one flat buffer that `.grad`
aliases, and gradient accumulation over several passes on top of that.

Bounds.  An accumulating call differs from the plain call plus the prior contents in the fp32 order of one addition, but two
clean runs of the same backward already differ: the norm backward adds its sums with fp32 atomics (DESIGN.md section 2).
Every tensor of a comparison is therefore bounded, as tests/test_gpu_poisoned_buffers.py bounds its training calls, by the
larger of 1e-6 relative L2 and twice the largest difference between two clean reference runs measured in the same test (a
per-tensor bound from one pair of runs proved too tight: one sample of the atomics' spread can be small by chance)."""

import pytest
import torch

from oracle import torch_oracle as O
from oracle import rew_end_training as RT

pytestmark = pytest.mark.gpu

REL = 1e-6


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _check(label, got, ref, again):
    """got / ref / again: lists of tensors; again is a second clean run of ref."""
    bound = max([REL] + [2 * _rel(a, r) for r, a in zip(ref, again)])
    worst = 0.0
    for k, (g, r) in enumerate(zip(got, ref)):
        e = _rel(g, r)
        worst = max(worst, e)
        assert torch.isfinite(g).all(), f"{label}: tensor {k} not finite"
        assert e <= bound, f"{label}: tensor {k} relative L2 {e:.3e} > {bound:.3e}"
    print(f"{label}: worst relative L2 {worst:.2e}, bound {bound:.2e}")


def _inner_cfg(name):
    if name == "default":
        return O.InnerCfg(), 2, 64
    if name == "wide":          # 128-channel levels: K-split wgrad blocks, and the split attention backward of the mid-block
        return O.InnerCfg(depths=[1, 1, 1, 1], channels=[64, 128, 128, 128]), 2, 64
    from oracle.make_golden import CASES

    return CASES["denoiser_small_heun"]["inner"], 3, 32   # 3 levels, attention inside the 64-channel level


def _denoiser(name, dev, seed=3):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.synthetic import randomize_module_

    i, b, hw = _inner_cfg(name)
    den = Denoiser(DenoiserConfig(InnerModelConfig(i.img_channels, i.num_steps_conditioning, i.cond_channels, list(i.depths),
                                                   list(i.channels), list(i.attn_depths), i.num_actions), 0.5, 0.3))
    randomize_module_(den.inner_model, seed)
    den = den.to(dev).train()
    sc = O.SigmaDistCfg()
    den.setup_training(SigmaDistributionConfig(sc.loc, sc.scale, sc.sigma_min, sc.sigma_max))
    return den, i, b, hw


def _rew_end_cfg(name):
    return O.RewEndCfg() if name == "default" else O.RewEndCfg(depths=[1, 1, 1, 1], channels=[128, 128, 128, 128])


def _rew_end(name, dev, seed=4):
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import randomize_module_

    c = _rew_end_cfg(name)
    m = RewEndModel(RewEndModelConfig(c.lstm_dim, c.img_channels, c.img_size, c.cond_channels, list(c.depths), list(c.channels),
                                      list(c.attn_depths), c.num_actions))
    randomize_module_(m, seed)
    return m.to(dev).train(), c


def _split(flat, layout):
    offs, nums = layout
    return [flat[o:o + n] for o, n in zip(offs, nums)]


# ------------------------------------------------------------------------------------------------ C ABI
class _DenoiserCalls:
    """dmd_inner_model_forward_train + dmd_denoiser_backward[_accumulate] through ctypes on one workspace, fixed inputs."""

    def __init__(self, name, dev):
        from diamond_b200 import _lib

        self.lib, self.L = _lib.lib(), _lib
        den, i, b, hw = _denoiser(name, dev)
        self.im = den.inner_model
        self.h = self.im.native()
        self.b, self.hw = b, hw
        g = torch.Generator().manual_seed(9)
        self.noisy = torch.randn(b, i.img_channels, hw, hw, generator=g).to(dev)
        self.cn = torch.randn(b, generator=g).to(dev)
        self.obs = torch.randn(b, i.num_steps_conditioning * i.img_channels, hw, hw, generator=g).to(dev)
        self.act = torch.randint(0, i.num_actions, (b, i.num_steps_conditioning), generator=g).to(dev)
        self.gout = torch.randn(b, i.img_channels, hw, hw, generator=g).to(dev)
        self.ws = torch.empty(self.lib.dmd_denoiser_train_workspace_bytes(self.h, b, hw, hw), dtype=torch.uint8, device=dev)
        self.out = torch.empty_like(self.noisy)
        offs, nums, self.total = self.im.grad_layout()
        self.layout = (offs, nums)
        self.no_grad_slots = [k for k, name in enumerate(self.im.state_dict()) if name == "noise_emb.weight"]

    def forward(self):
        self.L.check(self.lib.dmd_inner_model_forward_train(self.h, self.b, self.hw, self.hw, self.noisy.data_ptr(), self.cn.data_ptr(), 0,
                                                            self.obs.data_ptr(), self.act.data_ptr(), self.out.data_ptr(),
                                                            self.ws.data_ptr(), self.ws.numel(), self.L.current_stream()))

    def backward(self, accumulate, grads_ptr, numel):
        fn = self.lib.dmd_denoiser_backward_accumulate if accumulate else self.lib.dmd_denoiser_backward
        return fn(self.h, self.b, self.hw, self.hw, self.gout.data_ptr(), grads_ptr, numel, self.ws.data_ptr(), self.L.current_stream())


class _RewEndCalls:
    """dmd_rew_end_forward_train + dmd_rew_end_backward[_accumulate] through ctypes on one workspace, fixed inputs (with a carried
    state, so g_hx_in / g_cx_in are written too)."""

    def __init__(self, name, dev, b=4, t=5):
        from diamond_b200 import _lib

        self.lib, self.L = _lib.lib(), _lib
        self.m, c = _rew_end(name, dev)
        self.h = self.m._native()
        self.b, self.t = b, t
        g = torch.Generator().manual_seed(19)
        S, D = c.img_size, c.lstm_dim
        self.obs = torch.rand(b, t, c.img_channels, S, S, generator=g).to(dev) * 2 - 1
        self.nobs = torch.rand(b, t, c.img_channels, S, S, generator=g).to(dev) * 2 - 1
        self.act = torch.randint(0, c.num_actions, (b, t), generator=g).to(dev)
        self.hx, self.cx = (torch.randn(b, D, generator=g).to(dev) * 0.3 for _ in range(2))
        self.g_rew, self.g_end = torch.randn(b, t, 3, generator=g).to(dev), torch.randn(b, t, 2, generator=g).to(dev)
        self.g_hx, self.g_cx = torch.randn(b, D, generator=g).to(dev), torch.randn(b, D, generator=g).to(dev)
        self.outs = [torch.empty(b, t, 3, device=dev), torch.empty(b, t, 2, device=dev), torch.empty(b, D, device=dev),
                     torch.empty(b, D, device=dev)]
        self.g_in = [torch.empty(b, D, device=dev), torch.empty(b, D, device=dev)]
        self.ws = torch.empty(self.lib.dmd_rew_end_train_workspace_bytes(self.h, b, t), dtype=torch.uint8, device=dev)
        offs, nums, self.total = self.m.grad_layout()
        self.layout = (offs, nums)
        self.no_grad_slots = []

    def forward(self):
        self.L.check(self.lib.dmd_rew_end_forward_train(self.h, self.b, self.t, self.obs.data_ptr(), self.nobs.data_ptr(), self.act.data_ptr(),
                                                        self.hx.data_ptr(), self.cx.data_ptr(), *[o.data_ptr() for o in self.outs],
                                                        self.ws.data_ptr(), self.ws.numel(), self.L.current_stream()))

    def backward(self, accumulate, grads_ptr, numel):
        fn = self.lib.dmd_rew_end_backward_accumulate if accumulate else self.lib.dmd_rew_end_backward
        return fn(self.h, self.b, self.t, self.g_rew.data_ptr(), self.g_end.data_ptr(), self.g_hx.data_ptr(), self.g_cx.data_ptr(),
                  grads_ptr, numel, self.g_in[0].data_ptr(), self.g_in[1].data_ptr(), self.ws.data_ptr(), self.L.current_stream())


def _calls(model, net, dev):
    return _DenoiserCalls(net, dev) if model == "denoiser" else _RewEndCalls(net, dev)


@pytest.mark.parametrize("model,net", [("denoiser", "default"), ("denoiser", "wide"), ("rew_end", "default"), ("rew_end", "wide")])
def test_accumulate_entry_point_adds_the_plain_result(model, net):
    """Plain call twice (the run-to-run bound), the accumulating call on a seeded prefill, the plain call again.  The
    accumulating call launches exactly the kernels of the plain one, every tensor of its result is prefill + plain result,
    slots without a gradient keep the prefill, the plain call's result is unchanged by it, and g_hx_in / g_cx_in are the
    plain call's."""
    dev = _dev()
    c = _calls(model, net, dev)
    lib = c.lib

    def plain():
        grads = torch.full((c.total,), float("nan"), device=dev)
        c.forward()
        lib.dmd_launch_count(1)
        c.L.check(c.backward(False, grads.data_ptr(), c.total))
        n = lib.dmd_launch_count(0)
        torch.cuda.synchronize()
        return grads, n, [g.clone() for g in getattr(c, "g_in", [])]

    p1, n_plain, gin1 = plain()
    p2, _, _ = plain()
    g = torch.Generator().manual_seed(5)
    prefill = torch.cat([torch.randn(n, generator=g) * max(float(t.norm()) / max(n, 1) ** 0.5, 1e-3)
                         for t, n in zip(_split(p1.cpu(), c.layout), c.layout[1])])
    acc = torch.zeros(c.total, device=dev)
    for o, piece in zip(c.layout[0], torch.split(prefill, c.layout[1])):
        acc[o:o + piece.numel()] = piece.to(dev)
    before = acc.clone()
    c.forward()
    lib.dmd_launch_count(1)
    c.L.check(c.backward(True, acc.data_ptr(), c.total))
    n_acc = lib.dmd_launch_count(0)
    torch.cuda.synchronize()
    gin_acc = [x.clone() for x in getattr(c, "g_in", [])]
    p3, _, _ = plain()
    assert n_acc == n_plain, (n_acc, n_plain)
    pre = _split(before, c.layout)
    got = _split(acc, c.layout)
    ref = [a + b for a, b in zip(pre, _split(p1, c.layout))]
    again = [a + b for a, b in zip(pre, _split(p2, c.layout))]
    for k in c.no_grad_slots:
        assert torch.equal(got[k], pre[k]), "a slot without a gradient changed"
        ref[k], again[k] = pre[k], pre[k]
    _check(f"{model} {net} accumulate", got, ref, again)
    _check(f"{model} {net} plain after accumulate", _split(p3, c.layout), _split(p1, c.layout), _split(p2, c.layout))
    print(f"{model} {net}: plain result bit-identical before / after the accumulating call: {torch.equal(p1, p3)}; "
          f"two plain runs bit-identical: {torch.equal(p1, p2)}; {n_plain} launches")
    for a, b in zip(gin_acc, gin1):
        assert _rel(a, b) <= 1e-5


@pytest.mark.parametrize("model", ["denoiser", "rew_end"])
def test_accumulate_entry_point_rejects_bad_buffers_before_any_launch(model):
    dev = _dev()
    c = _calls(model, "default", dev)
    lib = c.lib
    grads = torch.zeros(c.total + 4, device=dev)
    c.forward()
    torch.cuda.synchronize()
    for ptr, numel, what in [(None, c.total, "null"), (grads.data_ptr(), c.total - 1, "too small"),
                             (grads.data_ptr() + 4, c.total, "16-byte aligned")]:
        lib.dmd_launch_count(1)
        assert c.backward(True, ptr, numel) != 0, what
        assert lib.dmd_launch_count(0) == 0, what
        print(what, "->", lib.dmd_last_error().decode())
    other = torch.zeros_like(c.ws)          # a workspace no forward_train ran on
    ws, c.ws = c.ws, other
    lib.dmd_launch_count(1)
    assert c.backward(True, grads.data_ptr(), c.total) != 0
    assert lib.dmd_launch_count(0) == 0
    c.ws = ws


# ------------------------------------------------------------------------------------------------ autograd
class _Batch:
    def __init__(self, obs, act, mask):
        self.obs, self.act, self.mask_padding = obs, act, mask


def _den_batch(i, b, hw, steps, seed, dev):
    g = torch.Generator().manual_seed(seed)
    T = i.num_steps_conditioning + steps
    obs = torch.randint(0, 256, (b, T, i.img_channels, hw, hw), generator=g).float().div(255).mul(2).sub(1).to(dev)
    act = torch.randint(0, i.num_actions, (b, T), generator=g).to(dev)
    return _Batch(obs, act, torch.ones(b, T, dtype=torch.bool, device=dev))


def _den_loss(den, batch, seed):
    torch.manual_seed(seed)
    return den(batch)[0]


def _aliases_last_flat_grad(model):
    flat = model.last_flat_grad
    offs, _, _ = model._grad_views_layout()
    return all(p.grad.data_ptr() == flat.data_ptr() + 4 * o for p, o in zip(model.parameters(), offs))


def test_denoiser_autoregressive_steps_accumulate_in_one_pass():
    """Denoiser.forward over 3 autoregressive steps (3 native nodes), one loss.backward(): `.grad` equals torch.autograd.grad of
    the same loss, and every `.grad` is the view of last_flat_grad at its dmd_denoiser_grad_layout offset."""
    dev = _dev()
    den, i, b, hw = _denoiser("small", dev)
    params = list(den.parameters())
    batch = _den_batch(i, b, hw, 3, 31, dev)
    ref = torch.autograd.grad(_den_loss(den, batch, 7), params)
    again = torch.autograd.grad(_den_loss(den, batch, 7), params)
    assert all(p.grad is None for p in params)            # torch.autograd.grad leaves .grad alone
    _den_loss(den, batch, 7).backward()
    torch.cuda.synchronize()
    _check("denoiser 3 autoregressive steps", [p.grad for p in params], ref, again)
    assert _aliases_last_flat_grad(den.inner_model)


def _acc_cycle_checks(label, model, params, loss_fn):
    """grad_acc_steps = 2 (each pass adopts its natively accumulated buffer by adding it to the `.grad`s the last one left),
    then zero_grad() (set to None: `.grad` is the pass's buffer again), zero_grad(set_to_none=False), a replaced .grad, and a
    native AdamW step (re-pack) followed by a new cycle.  loss_fn(k) is the loss of micro-batch k at the current weights."""
    from diamond_b200 import optim

    def refs(k):
        return torch.autograd.grad(loss_fn(k), params), torch.autograd.grad(loss_fn(k), params)

    (r0, a0), (r1, a1) = refs(0), refs(1)
    loss_fn(0).backward()
    loss_fn(1).backward()
    torch.cuda.synchronize()
    _check(f"{label} grad_acc_steps=2", [p.grad for p in params], [x + y for x, y in zip(r0, r1)], [x + y for x, y in zip(a0, a1)])
    model.zero_grad()
    loss_fn(1).backward()
    _check(f"{label} after zero_grad()", [p.grad for p in params], r1, a1)
    assert _aliases_last_flat_grad(model)
    model.zero_grad(set_to_none=False)
    loss_fn(0).backward()
    _check(f"{label} after zero_grad(set_to_none=False)", [p.grad for p in params], r0, a0)
    mine = torch.full_like(params[3], 0.25)
    params[3].grad = mine.clone()
    loss_fn(1).backward()
    want = [x + y for x, y in zip(r0, r1)]
    want_again = [x + y for x, y in zip(a0, a1)]
    want[3], want_again[3] = mine + r1[3], mine + a1[3]
    _check(f"{label} after a replaced .grad", [p.grad for p in params], want, want_again)
    opt = optim.AdamW(params, lr=1e-3)
    opt.step()                                                  # new weights: the next call re-packs
    opt.zero_grad()
    (s0, b0), (s1, b1) = refs(0), refs(1)
    loss_fn(0).backward()
    loss_fn(1).backward()
    torch.cuda.synchronize()
    _check(f"{label} new cycle after AdamW", [p.grad for p in params], [x + y for x, y in zip(s0, s1)], [x + y for x, y in zip(b0, b1)])


def test_denoiser_grad_acc_steps():
    dev = _dev()
    den, i, b, hw = _denoiser("small", dev)
    batches = [_den_batch(i, b, hw, 2, 40 + k, dev) for k in range(2)]
    _acc_cycle_checks("denoiser", den.inner_model, list(den.parameters()), lambda k: _den_loss(den, batches[k], 50 + k))


def _rew_end_batches(n, b, T, seed, dev):
    from test_gpu_rew_end_training import _batch, _seeded_batch

    raw = [_seeded_batch(b, T, seed + k) for k in range(n)]
    return raw, lambda k: _batch(*raw[k], dev)


def test_rew_end_grad_acc_steps():
    dev = _dev()
    m, _ = _rew_end("default", dev)
    _, batch = _rew_end_batches(2, 4, 6, 600, dev)
    _acc_cycle_checks("rew_end", m, list(m.parameters()), lambda k: m(batch(k))[0])


def test_rew_end_grad_acc_steps_at_trainer_shape_matches_oracle():
    """Two accumulated passes at the trainer's 32 x 19 against the fp32 oracle's summed gradient, within the bounds
    tests/test_gpu_rew_end_training.py uses for one pass."""
    from test_gpu_rew_end_training import PER_TENSOR_CAP

    dev = _dev()
    cfg = O.RewEndCfg()
    sd = O.seeded_state_dict(O.rew_end_shapes(cfg), 779)
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig

    m = RewEndModel(RewEndModelConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, cfg.cond_channels, list(cfg.depths),
                                      list(cfg.channels), list(cfg.attn_depths), cfg.num_actions))
    m.load_state_dict(sd)
    m = m.to(dev).train()
    raw, batch = _rew_end_batches(2, 32, 19, 1900, dev)
    for k in range(2):
        m(batch(k))[0].backward()
    torch.cuda.synchronize()
    torch.set_num_threads(16)
    ref = None
    for k in range(2):
        sdk = {n: v.clone().requires_grad_(True) for n, v in O.seeded_state_dict(O.rew_end_shapes(cfg), 779).items()}
        _, g = RT.rew_end_loss_grads_chunked(*raw[k], sdk, cfg, chunk=8)
        ref = g if ref is None else {n: ref[n] + g[n] for n in ref}
    grads = {n: p.grad.detach().cpu() for n, p in m.named_parameters()}
    num = den = 0.0
    rows = []
    for n in ref:
        d = grads[n].double() - ref[n].double()
        num += float(d.pow(2).sum()); den += float(ref[n].double().pow(2).sum())
        rows.append((float(d.norm() / ref[n].double().norm().clamp_min(1e-30)), n))
    whole = (num / den) ** 0.5
    print(f"rew_end 32x19 x 2 accumulated: whole-gradient rel {whole:.3e}, worst {sorted(rows, reverse=True)[:3]}")
    assert whole < 1e-3, whole
    for e, n in rows:
        assert e < PER_TENSOR_CAP, (n, e)


# ------------------------------------------------------------------------------------------------ poisoned buffers
@pytest.mark.parametrize("byte", [0x00, 0xFF, 0x5A], ids=lambda b: f"0x{b:02X}")
@pytest.mark.parametrize("model", ["denoiser", "rew_end"])
def test_accumulate_entry_point_on_poisoned_scratch(model, byte):
    """The training workspace before forward_train, the outputs and g_*_in start poisoned; the flat buffer is Kept (added to) and
    holds the prefill.  The result matches the same calls on clean memory."""
    from test_gpu_poisoned_buffers import poison_

    dev = _dev()
    c = _calls(model, "default", dev)

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
        return _split(acc, c.layout) + [x.clone() for x in getattr(c, "g_in", [])]

    ref, again = run(None), run(None)
    _check(f"{model} accumulate 0x{byte:02X}", run(byte), ref, again)
