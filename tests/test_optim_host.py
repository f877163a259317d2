"""CPU: the native optimizer's host side (diamond_b200/optim.py, dmd_grad_norm_clip / dmd_adamw_step argument checks) and the
float64 restatement of clip + AdamW (oracle/optim_reference.py) against torch's own optimizer.  No kernel launches: every C call
here fails its argument check, and the message names the check (on a machine without a GPU any CUDA call would fail with a
CUDA error instead)."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from diamond_b200 import _lib, optim
from oracle import make_reference_records as R
from oracle import optim_reference as OR
from oracle import torch_oracle as O


# ------------------------------------------------------------------------------------------------ Python-side rejections
@pytest.mark.parametrize("kw", [{"amsgrad": True}, {"maximize": True}, {"capturable": True}, {"differentiable": True},
                                {"fused": True}, {"fused": False}, {"foreach": True}, {"foreach": False}])
def test_adamw_rejects_torch_only_options(kw):
    with pytest.raises(ValueError, match=next(iter(kw))):
        optim.AdamW([torch.zeros(3)], lr=1e-4, **kw)


@pytest.mark.parametrize("make,match", [
    (lambda: torch.zeros(4), "CUDA"),
    (lambda: torch.zeros(4, dtype=torch.float64), "CUDA"),
    (lambda: torch.zeros(4, 4).t(), "CUDA"),
])
def test_adamw_rejects_cpu_params(make, match):
    with pytest.raises(ValueError, match=match):
        optim.AdamW([nn.Parameter(make())], lr=1e-4)


def test_adamw_rejects_tensor_and_invalid_hyperparameters():
    with pytest.raises(ValueError, match="lr"):
        optim.AdamW([torch.zeros(3)], lr=torch.tensor(1e-3))
    with pytest.raises(ValueError, match="learning rate"):
        optim.AdamW([torch.zeros(3)], lr=-1.0)
    with pytest.raises(ValueError, match="beta"):
        optim.AdamW([torch.zeros(3)], betas=(0.9, 1.0))


def test_clip_rejects_other_norms_and_foreach():
    p = nn.Parameter(torch.zeros(3))
    p.grad = torch.ones(3)
    for nt in (1.0, float("inf"), 3):
        with pytest.raises(ValueError, match="norm_type"):
            optim.clip_grad_norm_([p], 1.0, norm_type=nt)
    with pytest.raises(ValueError, match="foreach"):
        optim.clip_grad_norm_([p], 1.0, foreach=True)
    with pytest.raises(ValueError, match="CUDA"):
        optim.clip_grad_norm_([p], 1.0)


def test_clip_without_gradients_returns_zero():
    p = nn.Parameter(torch.zeros(3))
    assert float(optim.clip_grad_norm_([p], 1.0)) == 0.0


# ------------------------------------------------------------------------------------------------ C entry point checks
def _entries(n, **over):
    arr = (_lib.OptimTensor * n)()
    for i, e in enumerate(arr):
        e.param, e.grad, e.exp_avg, e.exp_avg_sq = 0x10000 + 64 * i, 0x20000 + 64 * i, 0x30000 + 64 * i, 0x40000 + 64 * i
        e.numel, e.weight_decay = 5 + i, 0.01
    for k, (i, v) in over.items():
        setattr(arr[i], k, v)
    return arr


def _err():
    return _lib.lib().dmd_last_error().decode()


def _clip(arr, n, max_norm=1.0, partial=0x50000, nbytes=1 << 20, out=0x60000):
    return _lib.lib().dmd_grad_norm_clip(arr, n, max_norm, 1, out, partial, nbytes, None)


def _adamw(arr, n, lr=1e-4, b1=0.9, b2=0.999, eps=1e-8, step=1.0):
    return _lib.lib().dmd_adamw_step(arr, n, lr, b1, b2, eps, step, None)


def test_c_checks_fail_before_any_cuda_call():
    lib = _lib.lib()
    cases = [
        (lambda: _clip(None, 1), "null tensor table"),
        (lambda: _adamw(None, 1), "null tensor table"),
        (lambda: _clip(_entries(2), 0), "n = 0"),
        (lambda: _adamw(_entries(2), -3), "n = -3"),
        (lambda: _clip(_entries(2, numel=(1, -1)), 2), "tensor 1 has negative numel"),
        (lambda: _adamw(_entries(2, numel=(0, -7)), 2), "tensor 0 has negative numel -7"),
        (lambda: _clip(_entries(3, grad=(2, None)), 3), "tensor 2 has a null grad"),
        (lambda: _adamw(_entries(2, exp_avg_sq=(0, None)), 2), "tensor 0 has a null param / exp_avg / exp_avg_sq"),
        (lambda: _adamw(_entries(2, param=(1, None)), 2), "tensor 1 has a null param"),
        (lambda: _clip(_entries(2, grad=(0, 0x20002)), 2), "grad pointer not 4-byte aligned"),
        (lambda: _adamw(_entries(2, weight_decay=(0, float("nan"))), 2), "weight_decay"),
        (lambda: _clip(_entries(2), 2, max_norm=float("nan")), "max_norm"),
        (lambda: _clip(_entries(2), 2, partial=None), "null partial"),
        (lambda: _clip(_entries(2), 2, out=None), "null norm_coef"),
        (lambda: _clip(_entries(2), 2, nbytes=8 * 1), "partial buffer too small"),
        (lambda: _clip(_entries(2), 2, partial=0x50004), "partial buffer not 8-byte aligned"),
        (lambda: _adamw(_entries(2), 2, lr=float("inf")), "lr"),
        (lambda: _adamw(_entries(2), 2, lr=float("nan")), "lr"),
        (lambda: _adamw(_entries(2), 2, eps=float("nan")), "eps"),
        (lambda: _adamw(_entries(2), 2, eps=float("-inf")), "eps"),
        (lambda: _adamw(_entries(2), 2, b2=1.0), "betas"),
        (lambda: _adamw(_entries(2), 2, step=0.0), "step"),
    ]
    for call, msg in cases:
        assert call() != 0, msg
        assert msg in _err(), (msg, _err())
    # a table that does not start on an 8-byte boundary
    buf = (C.c_char * (3 * C.sizeof(_lib.OptimTensor) + 16))()
    base = (C.addressof(buf) + 7) & ~7
    C.memmove(base + 4, C.addressof(_entries(2)), 2 * C.sizeof(_lib.OptimTensor))
    bad = C.cast(base + 4, C.POINTER(_lib.OptimTensor))
    assert _clip(bad, 2) != 0 and "misaligned tensor table" in _err()
    assert _adamw(bad, 2) != 0 and "misaligned tensor table" in _err()
    assert lib.dmd_grad_norm_partial_bytes(bad, 2) == 0 and "misaligned tensor table" in _err()


def test_partial_buffer_size_follows_the_chunking():
    lib = _lib.lib()
    arr = _entries(3, numel=(0, 1))
    arr[1].numel, arr[2].numel = 16384, 16385
    assert lib.dmd_grad_norm_partial_bytes(arr, 3) == 8 * (1 + 1 + 2)
    arr[0].numel = arr[1].numel = arr[2].numel = 0
    assert lib.dmd_grad_norm_partial_bytes(arr, 3) == 8   # nothing to reduce still gets one slot


# ------------------------------------------------------------------------------------------------ float64 restatement
def test_configure_opt_groups_restatement_matches_the_reference_split(golden_dir):
    """oracle.optim_reference.configure_opt_groups splits the denoiser the way the reference's utils.configure_opt did."""
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig

    inner = O.InnerCfg()
    den = Denoiser(DenoiserConfig(InnerModelConfig(inner.img_channels, inner.num_steps_conditioning, inner.cond_channels,
                                                   list(inner.depths), list(inner.channels), list(inner.attn_depths),
                                                   inner.num_actions), 0.5, 0.3))
    names = {id(p): n for n, p in den.named_parameters()}
    groups = OR.configure_opt_groups(den, 1e-2)
    got = [[names[id(p)] for p in g["params"]] for g in groups]
    assert got == [sorted(x) for x in R.load_records(golden_dir)["configure_opt_groups"]]
    assert [g["weight_decay"] for g in groups] == [1e-2, 0.0]


class _Mixed(nn.Module):
    """Every kind of parameter configure_opt sees, with numels that are not multiples of 4 and a 1-element tensor."""

    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 5, 3)
        self.norm = nn.GroupNorm(1, 5)
        self.emb = nn.Embedding(7, 3)
        self.lstm = nn.LSTMCell(6, 5)
        self.head = nn.Linear(5, 1)


@pytest.mark.parametrize("max_norm", [0.05, 1e3])
def test_oracle_reproduces_torch_adamw_and_clip_on_cpu(max_norm):
    """3 steps of clip_grad_norm_ + torch.optim.AdamW(foreach=False) with the configure_opt groups against the float64
    restatement: cumulative update within 1e-6 relative L2 (clip active at 0.05, inactive at 1e3)."""
    torch.manual_seed(0)
    model = _Mixed()
    p0 = [p.detach().clone() for p in model.parameters()]
    groups = OR.configure_opt_groups(model, 1e-2)
    opt = torch.optim.AdamW(groups, lr=1e-2, eps=1e-8, foreach=False)
    order = [p for g in groups for p in g["params"]]
    wds = [g["weight_decay"] for g in groups for _ in g["params"]]
    gen = torch.Generator().manual_seed(1)
    grads_per_step = []
    norms = []
    for _ in range(3):
        gs = [torch.randn(p.shape, generator=gen) * 0.1 for p in order]
        grads_per_step.append([g.clone() for g in gs])
        for p, g in zip(order, gs):
            p.grad = g
        norms.append(float(torch.nn.utils.clip_grad_norm_(order, max_norm)))
        opt.step()
    init ={id(p): q for p, q in zip(model.parameters(), p0)}
    start = [init[id(p)] for p in order]
    want, m, v = OR.train_steps(start, grads_per_step, wds, max_norm, 1e-2)
    num = sum(float(((p.detach().double() - w) ** 2).sum()) for p, w in zip(order, want))
    den = sum(float(((w - s.double()) ** 2).sum()) for w, s in zip(want, start))
    assert (num / den) ** 0.5 < 1e-6
    for p, mm, vv in zip(order, m, v):
        st = opt.state[p]
        for got, want in ((st["exp_avg"], mm), (st["exp_avg_sq"], vv)):   # fp32 moments: relative L2 at the fp32 level
            assert float((got.double() - want).norm() / want.norm()) < 1e-6
    g64 = [g.double() for g in grads_per_step[0]]
    assert abs(float(OR.clip_grad_norm(g64, max_norm)[1]) - norms[0]) <= 1e-6 * norms[0]
