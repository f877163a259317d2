"""Actor-critic: oracle pinned to the reference golden (CPU) and the native forward against it (GPU)."""
import os

import numpy as np
import pytest
import torch

from oracle import torch_oracle as O


def _inputs():
    rng = np.random.default_rng(91)
    b = 5
    obs = torch.from_numpy(rng.integers(0, 256, size=(3, b, 3, 64, 64)).astype(np.float32)).div(255).mul(2).sub(1)
    hx = torch.from_numpy(rng.standard_normal((b, 512)).astype(np.float32)) * 0.3
    cx = torch.from_numpy(rng.standard_normal((b, 512)).astype(np.float32)) * 0.3
    return obs, hx, cx


def test_oracle_actor_critic_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "actor_critic_default.npz"))
    cfg = O.ActorCriticCfg()
    sd = O.seeded_actor_critic_state_dict(cfg, 555)
    assert abs(O.state_checksum(sd) - float(g["weights_checksum"])) < 1e-6 * float(g["weights_checksum"])
    obs, hx, cx = _inputs()
    with torch.no_grad():
        for t in range(3):
            logits, val, (hx, cx) = O.predict_act_value(obs[t], hx, cx, sd, cfg)
            assert torch.allclose(logits, torch.from_numpy(g["logits"][t]), rtol=1e-5, atol=1e-5)
            assert torch.allclose(val, torch.from_numpy(g["val"][t]), rtol=1e-5, atol=1e-5)
    assert torch.allclose(hx, torch.from_numpy(g["hx"]), atol=1e-5) and torch.allclose(cx, torch.from_numpy(g["cx"]), atol=1e-5)


def test_actor_critic_mirror_state_dict_and_init():
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig

    cfg = O.ActorCriticCfg()
    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    assert [(k, tuple(v.shape)) for k, v in ac.state_dict().items()] == O.actor_critic_shapes(cfg)
    assert sum(p.numel() for p in ac.parameters()) == 3_229_637  # BASELINE.md
    assert float(ac.actor_linear.weight.abs().sum()) == 0 and float(ac.critic_linear.weight.abs().sum()) == 0
    assert torch.all(ac.lstm.bias_ih[512:1024] == 1) and float(ac.lstm.bias_hh.abs().sum()) == 0
    with pytest.raises(RuntimeError):  # no CPU route: the native executor refuses non-CUDA parameters
        ac.predict_act_value(torch.zeros(1, 3, 64, 64), (torch.zeros(1, 512), torch.zeros(1, 512)))


@pytest.mark.gpu
def test_native_actor_critic_matches_reference_golden(golden_dir):
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig

    dev = torch.device("cuda:0")
    g = np.load(os.path.join(golden_dir, "actor_critic_default.npz"))
    cfg = O.ActorCriticCfg()
    sd = O.seeded_actor_critic_state_dict(cfg, 555)
    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    ac.load_state_dict(sd)
    ac = ac.to(dev).eval()
    obs, hx, cx = _inputs()
    hx, cx = hx.to(dev), cx.to(dev)

    def rel(a, b):
        return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt())

    with torch.no_grad():
        for t in range(3):
            out = ac.predict_act_value(obs[t].to(dev), (hx, cx))
            hx, cx = out.hx_cx
            e1, e2 = rel(out.logits_act.cpu(), torch.from_numpy(g["logits"][t])), rel(out.val.cpu(), torch.from_numpy(g["val"][t]))
            print(f"step {t}: logits rel err {e1:.3e}  value rel err {e2:.3e}")
            # logits / hidden state: 1e-3.  The scalar value head is a single 512-term dot product with cancellation
            # (|val| << sum|w_i h_i|), so its relative error over 5 numbers is bounded at 2e-3.
            assert e1 < 1e-3 and e2 < 2e-3
    assert rel(hx.cpu(), torch.from_numpy(g["hx"])) < 1e-3 and rel(cx.cpu(), torch.from_numpy(g["cx"])) < 1e-3
    # sub-batch consistency (dead-env path calls predict_act_value on a subset, env_loop.py:49)
    with torch.no_grad():
        full = ac.predict_act_value(obs[0].to(dev), (hx, cx))
        part = ac.predict_act_value(obs[0][1:3].to(dev), (hx[1:3], cx[1:3]))
    assert torch.allclose(full.logits_act[1:3], part.logits_act, atol=1e-5)


@pytest.mark.gpu
def test_native_actor_critic_rejects_parameters_that_are_not_contiguous_fp32():
    """The native layer reads every parameter through a raw fp32 pointer: a transposed or fp64 parameter is refused, as the
    denoiser and the reward / termination model refuse it, and the same model runs once the parameter is restored."""
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig

    dev = torch.device("cuda:0")
    cfg = O.ActorCriticCfg()
    ac = ActorCritic(ActorCriticConfig(cfg.lstm_dim, cfg.img_channels, cfg.img_size, list(cfg.channels), list(cfg.down), cfg.num_actions))
    ac = ac.to(dev).eval()
    obs = torch.zeros(2, cfg.img_channels, cfg.img_size, cfg.img_size, device=dev)
    hx = cx = torch.zeros(2, cfg.lstm_dim, device=dev)
    for p, bad in ((ac.lstm.weight_hh, lambda d: d.t().contiguous().t()), (ac.critic_linear.bias, lambda d: d.double())):
        good = p.data
        p.data = bad(good)
        with torch.no_grad(), pytest.raises(RuntimeError, match="contiguous fp32"):
            ac.predict_act_value(obs, (hx, cx))
        p.data = good
        with torch.no_grad():
            ac.predict_act_value(obs, (hx, cx))


def test_accumulated_native_gradients_are_adopted_like_accumulate_grad():
    """Host half of the BPTT gradient path (CPU): the flat buffer the native backward nodes accumulated into becomes `.grad` of
    every trainable parameter as a VIEW (so one all-reduce on the buffer averages the model), frozen parameters are skipped, and
    a second backward pass ADDS to the existing `.grad` (what autograd's AccumulateGrad does).  The native half (the nodes adding
    into the buffer) is exercised on the GPU by tests/test_gpu_training.py::test_actor_critic_training_step_matches_reference."""
    from diamond_b200.models.actor_critic import ActorCritic, ActorCriticConfig

    ac = ActorCritic(ActorCriticConfig(64, 3, 16, [32, 32], [1, 1], 4))
    names = list(ac.state_dict().keys())
    sizes = [v.numel() for v in ac.state_dict().values()]
    offs, o = [], 0
    for n in sizes:                      # the layout dmd_actor_critic_grad_layout reports: state_dict order, 16-byte aligned slices
        offs.append(o)
        o += (n + 3) // 4 * 4
    ac.grad_layout = lambda: (offs, sizes, o)          # stands in for the C-ABI query (needs the CUDA library)
    frozen = next(iter(ac.parameters()))
    frozen.requires_grad_(False)
    flat = torch.arange(o, dtype=torch.float32)
    ac.__dict__["_grad_acc"] = flat
    ac._adopt_accumulated_grads()
    assert "_grad_acc" not in ac.__dict__ and ac.last_flat_grad is flat
    index = {k: i for i, k in enumerate(names)}
    for k, p in ac.named_parameters():
        if p is frozen:
            assert p.grad is None
            continue
        want = flat[offs[index[k]]:offs[index[k]] + sizes[index[k]]].view_as(p)
        assert torch.equal(p.grad, want) and p.grad.data_ptr() == want.data_ptr()
    first = {k: p.grad.clone() for k, p in ac.named_parameters() if p.grad is not None}
    ac.__dict__["_grad_acc"] = torch.ones(o)
    ac._adopt_accumulated_grads()
    for k, p in ac.named_parameters():
        if p.grad is not None:
            assert torch.equal(p.grad, first[k] + 1)
    ac._adopt_accumulated_grads()        # nothing pending: a no-op
