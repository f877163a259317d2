"""CPU, two gloo ranks: the native models' gradients under torch DistributedDataParallel with its default arguments (the
reference trainer wraps every model in `DDP(module)`, utils.py:105-106), and its find_unused_parameters, gradient_as_bucket_view
and no_sync variants.

The stand-in native module of tests/test_grad_accumulation_host.py runs the real NativeStateMixin code with a CPU function in
place of the native backward; here its forward also records, as the native autograd Functions do, whether it runs inside a
DDP forward.  Every rank trains on its own input, so the rank mean differs from each local gradient.  All values are small
multiples of 0.5: DDP's division by the world size and its sum are exact, and `.grad` must equal the rank mean exactly.  The
native GPU models run the same checks in tests/test_gpu_ddp.py."""
import datetime
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
from torch.nn.parallel import DistributedDataParallel as DDP

from test_grad_accumulation_host import _Toy as _HostToy, _ToyFn, _aliases_flat

WORLD = 2


class _DDPToyFn(_ToyFn):
    @staticmethod
    def forward(ctx, module, x, *params):
        ctx.under_ddp = module._under_ddp()
        return _ToyFn.forward(ctx, module, x, *params)


class _Toy(_HostToy):
    def forward(self, x):
        return _DDPToyFn.apply(self, x, *self.parameters())


class _Steps(nn.Module):
    """A wrapper that owns the native module and calls it several times per forward, as Denoiser.forward calls its InnerModel
    once per autoregressive step: y = x_0 + 2 x_1 + x_2 ... with x_k the k-th call."""

    def __init__(self, n):
        super().__init__()
        self.inner, self.n = _Toy(), n

    def forward(self, x):
        return sum((1 + (k % 2)) * self.inner(x) for k in range(self.n))


def _s(n, x):
    """The stand-in's gradient scale for `_Steps(n)` on input x (one element)."""
    return sum(1 + (k % 2) for k in range(n)) * x


def _want(model, s):
    return [torch.full_like(p, (k + 1) * s) for k, p in enumerate(model.parameters())]


def _grads_are(model, s):
    return all(p.grad is not None and torch.equal(p.grad, w) for p, w in zip(model.parameters(), _want(model, s)))


def _rank_mean(f):
    return sum(f(r) for r in range(WORLD)) / WORLD


def _case_steps(rank, n, iters=2, **ddp_kwargs):
    """`iters` iterations of forward, backward, check, zero_grad through DDP(_Steps(n)) (n = 1: DDP around the native module
    itself), the input changing every iteration."""
    wrapper = _Steps(n)
    m = wrapper.inner
    ddp = DDP(m if n == 1 else wrapper, **ddp_kwargs)
    bad = []
    for it in range(iters):
        x = torch.tensor([1.0 + rank + it])
        ddp(x).sum().backward()
        if not _grads_are(m, _rank_mean(lambda r: _s(n, 1.0 + r + it))):
            bad.append(f"iteration {it}: .grad {[p.grad.flatten()[0].item() for p in m.parameters()]}")
        calls = [a for a, _ in m.calls[-n:]]
        if calls != [False] + [True] * (n - 1):
            bad.append(f"iteration {it}: native calls {calls}")
        if m.last_flat_grad is not m.calls[-1][1] or "_grad_acc" in m.__dict__ or "_grad_views" in m.__dict__:
            bad.append(f"iteration {it}: pass buffer not handed on")
        m.zero_grad()
    return bad


def _case_grad_acc_steps(rank):
    """grad_acc_steps = 2: two passes before the optimizer step, each all-reduced (as the reference trainer does)."""
    m = _Toy()
    ddp = DDP(m)
    for k in range(2):
        ddp(torch.tensor([1.0 + rank + k])).sum().backward()
    want = _rank_mean(lambda r: 1.0 + r) + _rank_mean(lambda r: 2.0 + r)
    return [] if _grads_are(m, want) else [f".grad {[p.grad.flatten()[0].item() for p in m.parameters()]}, want {want}"]


def _case_no_sync(rank):
    """Under no_sync() every rank keeps its local gradient; the next synchronised pass averages the accumulated sum."""
    wrapper = _Steps(2)
    m = wrapper.inner
    ddp = DDP(wrapper)
    bad = []
    with ddp.no_sync():
        ddp(torch.tensor([1.0 + rank])).sum().backward()
    if not _grads_are(m, _s(2, 1.0 + rank)):
        bad.append(f"no_sync: .grad {[p.grad.flatten()[0].item() for p in m.parameters()]}")
    ddp(torch.tensor([1.0 + rank])).sum().backward()
    if not _grads_are(m, 2 * _rank_mean(lambda r: _s(2, 1.0 + r))):
        bad.append(f"after no_sync: .grad {[p.grad.flatten()[0].item() for p in m.parameters()]}")
    return bad


def _case_outside_ddp(rank):
    """A native module that a DDP-wrapped module calls without owning it (as the actor-critic's rollout calls the world model)
    and the same module called directly after DDP use: both keep the local gradient, adopted at the end of the pass as a
    view of one flat buffer."""
    m = _Toy()

    class Caller(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.ones(1))

        def forward(self, x):
            return self.w * m(x)
    caller = DDP(Caller())
    bad = []
    caller(torch.tensor([1.0 + rank])).sum().backward()
    if not (_grads_are(m, 1.0 + rank) and _aliases_flat(m)):
        bad.append("called inside another module's DDP forward")
    inner = _Toy()
    DDP(inner)(torch.tensor([1.0 + rank])).sum().backward()
    inner.zero_grad()
    (inner(torch.tensor([1.0 + rank])) + inner(torch.tensor([1.0 + rank]))).sum().backward()
    if not (_grads_are(inner, 2 * (1.0 + rank)) and _aliases_flat(inner) and [a for a, _ in inner.calls[-2:]] == [False, True]):
        bad.append("called directly after DDP use")
    return bad


CASES = {
    "one_node": lambda r: _case_steps(r, 1),
    "three_nodes": lambda r: _case_steps(r, 3),
    "grad_acc_steps": _case_grad_acc_steps,
    "find_unused_parameters": lambda r: _case_steps(r, 3, find_unused_parameters=True),
    "gradient_as_bucket_view": lambda r: _case_steps(r, 3, gradient_as_bucket_view=True),
    "no_sync": _case_no_sync,
    "outside_ddp": _case_outside_ddp,
}


def _worker(rank, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=WORLD, timeout=datetime.timedelta(seconds=60))
    out = {}
    for name, case in CASES.items():
        try:
            out[name] = case(rank)
        except Exception as e:      # noqa: BLE001 -- reported per case; the collectives of later cases still pair up
            out[name] = [repr(e)]
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def results():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, port, q)) for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        out = dict(q.get(timeout=240) for _ in range(WORLD))
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_ddp_gradients_are_the_rank_mean(results, case):
    for rank in range(WORLD):
        assert results[rank][case] == [], (rank, results[rank][case])
