"""CPU: the host half of native gradient accumulation for the denoiser and the reward / termination model.

A stand-in module replaces the native backward by a CPU function with the same contract (write or ADD every parameter gradient
into one flat buffer at the layout offsets); everything else -- which call each node of a backward pass makes, when `.grad` is
adopted, what `last_flat_grad` names, deepcopy, the single all-reduce -- is the code InnerModel and RewEndModel run.  The native half is
exercised on the GPU by tests/test_gpu_grad_accumulation.py."""
import copy
import ctypes
import os
import re
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from diamond_b200 import _lib
from diamond_b200.utils import NativeStateMixin, allreduce_native_gradients

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Toy(NativeStateMixin, nn.Module):
    """Three parameters and a buffer, laid out like a native model: state_dict order, 16-byte slices.
    `calls` records (accumulate, buffer) of every stand-in native backward."""

    def __init__(self):
        super().__init__()
        self.a = nn.Parameter(torch.zeros(3, 2))
        self.register_buffer("noise", torch.zeros(5))   # a slot without a gradient, like noise_emb.weight
        self.b = nn.Parameter(torch.zeros(5))
        self.c = nn.Parameter(torch.zeros(2, 2))
        self.calls = []

    @property
    def device(self):
        return self.a.device

    def grad_layout(self):
        offs, nums, o = [], [], 0
        for v in self.state_dict().values():
            offs.append(o)
            nums.append(v.numel())
            o += (v.numel() + 3) // 4 * 4
        return offs, nums, o

    def forward(self, x):
        return _ToyFn.apply(self, x, *self.parameters())


class _ToyFn(torch.autograd.Function):
    """y = x * (sum a + 2 sum b + 3 sum c): d/dp of sum(w * y) is (k * sum(w * x)) for every element of parameter k."""

    @staticmethod
    def forward(ctx, module, x, *params):
        ctx.module, ctx.x = module, x
        return x * sum((k + 1) * p.sum() for k, p in enumerate(params))

    @staticmethod
    def backward(ctx, g):
        module = ctx.module
        s = float((g * ctx.x).sum())

        def run(flat, accumulate):
            module.calls.append((accumulate, flat))
            offs, nums, _ = module._grad_views_layout()
            if not accumulate:
                flat.zero_()
            for k, (o, n) in enumerate(zip(offs, nums)):
                flat[o:o + n] += (k + 1) * s
        return (None, None, *module._native_param_grads(ctx, run))


def _want(model, s):
    return [torch.full_like(p, (k + 1) * s) for k, p in enumerate(model.parameters())]


def _aliases_flat(model):
    flat = model.last_flat_grad
    offs, nums, _ = model._grad_views_layout()
    return all(p.grad.data_ptr() == flat.data_ptr() + 4 * o and p.grad.shape == p.shape
               for p, o in zip(model.parameters(), offs) if p.requires_grad)


def _check(model, s):
    for p, w in zip(model.parameters(), _want(model, s)):
        assert torch.equal(p.grad, w), (p.grad, w)


def test_nodes_of_one_pass_add_into_one_buffer():
    m = _Toy()
    x = torch.tensor([1.0, 2.0])
    (m(x) + 2 * m(x) + m(x)).sum().backward()     # three nodes in one pass (autoregressive steps): s = 3 + 6 + 3
    assert [a for a, _ in m.calls] == [False, True, True]
    assert m.calls[0][1] is m.calls[1][1] is m.calls[2][1] is m.last_flat_grad
    assert "_grad_acc" not in m.__dict__
    _check(m, 12.0)
    assert _aliases_flat(m)


def test_later_passes_add_to_the_grads_tensor_by_tensor():
    """grad_acc_steps > 1: every pass fills its own buffer and adds it to the existing `.grad`s, as AccumulateGrad does;
    `last_flat_grad` names the last pass's buffer, which the `.grad`s then do not alias."""
    m = _Toy()
    x = torch.tensor([1.0, 2.0])
    (m(x) + m(x)).sum().backward()
    first = m.last_flat_grad
    m(x).sum().backward()
    assert [a for a, _ in m.calls] == [False, True, False]
    assert m.calls[2][1] is m.last_flat_grad is not first
    _check(m, 9.0)
    assert not _aliases_flat(m)                    # allreduce_native_gradients then takes its bucketed path


def test_zero_grad_set_to_none_starts_from_nothing():
    m = _Toy()
    x = torch.tensor([1.0, 1.0])
    m(x).sum().backward()
    old = m.last_flat_grad
    m.zero_grad()                                  # torch >= 2.0 default: set_to_none=True
    m(3 * x).sum().backward()
    assert [a for a, _ in m.calls] == [False, False]
    _check(m, 6.0)                                 # nothing stale from the first pass
    assert _aliases_flat(m) and m.last_flat_grad is not old


def test_zero_grad_in_place_keeps_values_right():
    m = _Toy()
    x = torch.tensor([1.0, 1.0])
    m(x).sum().backward()
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    opt.zero_grad(set_to_none=False)
    m(x).sum().backward()
    _check(m, 2.0)


def test_replaced_grad_is_added_to():
    m = _Toy()
    x = torch.tensor([1.0])
    m(x).sum().backward()
    m.zero_grad()
    m.b.grad = torch.full_like(m.b, 100.0)         # the caller sets one .grad
    m(x).sum().backward()
    assert torch.equal(m.a.grad, torch.full_like(m.a, 1.0))
    assert torch.equal(m.b.grad, torch.full_like(m.b, 102.0))
    assert torch.equal(m.c.grad, torch.full_like(m.c, 3.0))


def test_frozen_parameter_is_skipped():
    m = _Toy()
    m.b.requires_grad_(False)
    x = torch.tensor([1.0])
    (m(x) + m(x)).sum().backward()
    assert [a for a, _ in m.calls] == [False, True]
    assert m.b.grad is None
    assert torch.equal(m.a.grad, torch.full_like(m.a, 2.0)) and torch.equal(m.c.grad, torch.full_like(m.c, 6.0))
    assert _aliases_flat(m)


def test_autograd_grad_returns_gradients_and_leaves_grad_alone():
    m = _Toy()
    x = torch.tensor([1.0, 2.0])
    m(x).sum().backward()
    before = [p.grad.clone() for p in m.parameters()]
    gs = torch.autograd.grad((m(x) + m(x)).sum(), list(m.parameters()))
    assert [a for a, _ in m.calls] == [False, False, False]   # every node writes its own buffer
    for g, w in zip(gs, _want(m, 6.0)):
        assert torch.equal(g, w)
    for p, b in zip(m.parameters(), before):
        assert torch.equal(p.grad, b)
    # and loss.backward() afterwards still adds to the .grads it left alone
    m(x).sum().backward()
    _check(m, 6.0)


def test_backward_with_inputs_subset_goes_through_autograd():
    m = _Toy()
    x = torch.tensor([1.0])
    m(x).sum().backward(inputs=[m.a])
    assert [a for a, _ in m.calls] == [False]
    assert torch.equal(m.a.grad, torch.full_like(m.a, 1.0)) and m.b.grad is None and m.c.grad is None


def test_pass_that_died_does_not_leak_into_the_next():
    m = _Toy()
    x = torch.tensor([1.0])

    class Boom(torch.autograd.Function):
        @staticmethod
        def forward(ctx, y):
            return y.clone()

        @staticmethod
        def backward(ctx, g):
            raise ValueError("boom")
    y = Boom.apply(m(x)) + m(x)                    # the plain node of m runs first, then Boom raises
    try:
        y.sum().backward()
    except ValueError:
        pass
    m.zero_grad()
    m(x).sum().backward()
    assert m.calls[-1][0] is False
    _check(m, 1.0)
    assert "_grad_acc" not in m.__dict__


def test_deepcopy_and_pickle_drop_the_buffers():
    m = _Toy()
    x = torch.tensor([1.0])
    m(x).sum().backward()
    m.__dict__["_grad_acc"] = torch.zeros(4)
    for k in ("_grad_acc", "_grad_task", "last_flat_grad"):
        assert k in m.__dict__
    c = copy.deepcopy(m)
    for k in ("_grad_acc", "_grad_task", "last_flat_grad"):
        assert k not in c.__dict__ and k not in m.__getstate__()


# ---------------------------------------------------------------------------------------------- C ABI

def _header_decl(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "diamond_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\);", text)
    assert m, name
    return [re.sub(r"\s+", " ", a.strip()) for a in m.group(1).split(",")]


def test_accumulate_entry_points_have_their_twins_signatures():
    for twin in ("dmd_denoiser_backward", "dmd_rew_end_backward"):
        acc = twin + "_accumulate"
        assert _header_decl(acc) == _header_decl(twin)
        assert _lib.SIGNATURES[acc] == _lib.SIGNATURES[twin]
        assert hasattr(ctypes.CDLL(_lib.LIB_PATH), acc)


# ---------------------------------------------------------------------------------------------- one collective per step

def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    m = _Toy()
    x = torch.tensor([1.0 + rank])
    (m(x) + m(x)).sum().backward()                 # two autoregressive steps in one pass: s = 2 (1 + rank)
    calls = allreduce_native_gradients(m)
    mean_s = sum(2.0 * (1 + r) for r in range(world)) / world
    ok = all(torch.equal(p.grad, w) for p, w in zip(m.parameters(), _want(m, mean_s))) and _aliases_flat(m)
    q.put((rank, calls, ok))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_autoregressive_gradients_are_one_collective():
    """Before native accumulation, the second node's buffer became last_flat_grad while the .grads kept the first: bucketed."""
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = sorted(q.get(timeout=180) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, calls, ok in out:
        assert calls == 1 and ok
