"""GPU, two ranks: the denoiser, the reward/termination model and the actor-critic trained under torch
DistributedDataParallel with its default arguments, wrapped as the reference trainer wraps them (`DDP(module)`,
utils.py:105-106).

Each rank trains on its own data.  With torch.use_deterministic_algorithms(True) the native backward is bit-reproducible, so
a rank first computes its local gradient without DDP and then the same step through the wrapper.  DDP divides each rank's
gradient by the world size (exact) and sums two fp32 terms, so `.grad` must equal the mean of the all-gathered local
gradients bit for bit.  After clip_grad_norm_ and torch.optim.AdamW the parameters are identical on both ranks; a second
step, at the stepped weights, repeats every check.

Two ranks share one device over gloo (which all-reduces and broadcasts CUDA tensors); with two visible devices, two ranks on
two devices over NCCL run too.  The CPU half, with the find_unused_parameters, gradient_as_bucket_view and no_sync variants,
is tests/test_ddp_host.py."""
import datetime
import os
import random
import socket
import types

# torch's own cuBLAS calls refuse deterministic mode without a fixed workspace configuration; it is read when cuBLAS starts
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import pytest  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

pytestmark = pytest.mark.gpu

WORLD = 2
STEPS = 2
MODELS = ("denoiser", "rew_end", "actor_critic")


# ------------------------------------------------------------------------------------------------ models and losses
# Each builder returns (module DDP wraps, loss(callable, rank, step)).  The loss of (rank, step) draws the same data and the
# same random numbers every time it is called: the local pass and the DDP pass of a step see identical inputs.

def _denoiser(dev):
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, InnerModelConfig, SigmaDistributionConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [1, 1, 1, 1], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    den = den.to(dev).train()
    den.setup_training(SigmaDistributionConfig(-0.4, 1.2, 2e-3, 20))

    def loss(model, rank, step):
        obs, act, _ = frame_stacks(2, 4 + 2, 3, 64, 64, 4, 100 * rank + step)   # 2 autoregressive steps
        batch = types.SimpleNamespace(obs=obs.to(dev), act=act.to(dev), mask_padding=torch.ones(2, 6, dtype=torch.bool, device=dev))
        torch.manual_seed(10 * rank + step)       # sigma, offset noise and white noise of every step
        return model(batch)[0]
    return den, loss


def _rew_end(dev):
    import test_gpu_rew_end_training as TR
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import randomize_module_

    m = RewEndModel(RewEndModelConfig(512, 3, 64, 128, [1, 1, 1, 1], [32] * 4, [0] * 4, 4))
    randomize_module_(m, 2025)
    m = m.to(dev).train()

    def loss(model, rank, step):
        return model(TR._batch(*TR._seeded_batch(4, 6, 300 + 10 * rank + step), dev))[0]   # some segments die mid-way
    return m, loss


def _actor_critic(dev):
    from diamond_b200.envs import WorldModelEnv, WorldModelEnvConfig
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig, ActorCriticLossConfig
    from diamond_b200.models.diffusion import Denoiser, DenoiserConfig, DiffusionSamplerConfig, InnerModelConfig
    from diamond_b200.models.rew_end_model import RewEndModel, RewEndModelConfig
    from diamond_b200.synthetic import frame_stacks, randomize_module_

    den = Denoiser(DenoiserConfig(InnerModelConfig(3, 4, 256, [1, 1, 1, 1], [64] * 4, [0] * 4, 4), 0.5, 0.3))
    randomize_module_(den.inner_model, 2024)
    rem = RewEndModel(RewEndModelConfig(512, 3, 64, 128, [1, 1, 1, 1], [32] * 4, [0] * 4, 4))
    randomize_module_(rem, 2025)
    ac = ActorCritic(ActorCriticConfig(512, 3, 64, [32, 32, 64, 64], [1, 1, 1, 1], 4))
    randomize_module_(ac, 2026)
    den, rem, ac = den.to(dev).eval(), rem.to(dev).eval(), ac.to(dev).train()
    envs = 4

    def loss(model, rank, step):
        """One update of 6 imagined steps from a fresh WorldModelEnv (episodes of 4 steps: one reset and burn-in inside)."""
        pool = [frame_stacks(envs, 4, 3, 64, 64, 4, 1000 * rank + 10 * step + k)[:2] for k in range(2)]

        class Loader:
            batch_sampler = types.SimpleNamespace(batch_size=envs)

            def __iter__(self):
                k = 0
                while True:
                    obs, act = pool[k % len(pool)]
                    k += 1
                    yield types.SimpleNamespace(obs=obs, act=act)
        random.seed(rank * 7 + step)
        torch.manual_seed(rank * 7 + step)
        ac.env_loop = ac.loss_cfg = None
        ac.setup_training(WorldModelEnv(den, rem, Loader(), WorldModelEnvConfig(4, 2, DiffusionSamplerConfig(3))),
                          ActorCriticLossConfig(6, 0.985, 0.95, 1.0, 0.001))
        return model()[0]
    return ac, loss


BUILDERS = {"denoiser": _denoiser, "rew_end": _rew_end, "actor_critic": _actor_critic}


# ------------------------------------------------------------------------------------------------ one rank
def _flat(ts):
    return torch.cat([t.detach().reshape(-1).cpu() for t in ts])


def _train(name, rank, dev):
    """STEPS optimizer steps of one model through DDP; returns the problems found."""
    from torch.nn.parallel import DistributedDataParallel as DDP

    module, loss = BUILDERS[name](dev)
    params = [p for p in module.parameters() if p.requires_grad]
    ddp = DDP(module)
    opt = torch.optim.AdamW(params, lr=1e-3)
    bad = []
    for step in range(STEPS):
        opt.zero_grad()
        local_loss = loss(module, rank, step)
        local_loss.backward()
        local = _flat(p.grad for p in params)
        opt.zero_grad()
        ddp_loss = loss(ddp, rank, step)
        ddp_loss.backward()
        got = _flat(p.grad for p in params)
        gathered = [None] * WORLD
        dist.all_gather_object(gathered, local)
        mean = sum(g / WORLD for g in gathered)           # DDP: every rank's gradient divided by the world size, then summed
        if not torch.equal(local_loss.detach().cpu(), ddp_loss.detach().cpu()):
            bad.append(f"step {step}: loss {float(ddp_loss)} through DDP, {float(local_loss)} without")
        if torch.equal(gathered[0], gathered[1]):
            bad.append(f"step {step}: both ranks have the same local gradient; the check would not see a missing average")
        if not torch.equal(got, mean):
            d = (got - mean).abs()
            bad.append(f"step {step}: .grad differs from the rank mean in {int((d > 0).sum())} of {d.numel()} elements "
                       f"(largest {float(d.max()):.3e}, mean |grad| {float(mean.abs().mean()):.3e})")
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()
        weights = [None] * WORLD
        dist.all_gather_object(weights, _flat(params))
        if not torch.equal(weights[0], weights[1]):
            bad.append(f"step {step}: parameters differ between the ranks after AdamW")
    return bad


def _worker(rank, backend, per_rank_device, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank if per_rank_device else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=WORLD, timeout=datetime.timedelta(seconds=180))
    torch.use_deterministic_algorithms(True)
    out = {}
    for name in MODELS:
        try:
            out[name] = _train(name, rank, dev)
        except Exception as e:      # noqa: BLE001 -- reported per model
            out[name] = [f"{type(e).__name__}: {e}"]
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def _run(backend, per_rank_device):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, backend, per_rank_device, port, q)) for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        out = dict(q.get(timeout=900) for _ in range(WORLD))
        for p in procs:
            p.join(timeout=120)
    finally:
        for p in procs:          # nothing outlives the test
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return out


@pytest.fixture(scope="module")
def gloo_one_device():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return _run("gloo", False)


@pytest.fixture(scope="module")
def nccl_two_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    return _run("nccl", True)


@pytest.mark.parametrize("name", MODELS)
def test_ddp_two_ranks_one_device_gloo(gloo_one_device, name):
    for rank in range(WORLD):
        assert gloo_one_device[rank][name] == [], (rank, gloo_one_device[rank][name])


@pytest.mark.parametrize("name", MODELS)
def test_ddp_two_ranks_two_devices_nccl(nccl_two_devices, name):
    for rank in range(WORLD):
        assert nccl_two_devices[rank][name] == [], (rank, nccl_two_devices[rank][name])
