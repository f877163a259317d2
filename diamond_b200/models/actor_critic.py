"""ActorCritic (reference: src/models/actor_critic.py) with a native sm_90a forward for predict_act_value."""
import math
from collections import namedtuple
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from torch.distributions.categorical import Categorical

from .. import _lib
from ..coroutines.env_loop import make_env_loop
from ..utils import LossAndLogs, NativeStateMixin, init_lstm
from .blocks import SmallResBlock, _NativeOnly, conv3x3

ActorCriticOutput = namedtuple("ActorCriticOutput", "logits_act val hx_cx")


@dataclass
class ActorCriticLossConfig:  # actor_critic.py:21-27
    backup_every: int
    gamma: float
    lambda_: float
    weight_value_loss: float
    weight_entropy_loss: float


@dataclass
class ActorCriticConfig:  # actor_critic.py:30-37
    lstm_dim: int
    img_channels: int
    img_size: int
    channels: List[int]
    down: List[int]
    num_actions: Optional[int] = None


class ActorCriticEncoder(_NativeOnly):  # actor_critic.py:101-113 (parameter container; executed natively)
    def __init__(self, cfg: ActorCriticConfig) -> None:
        super().__init__()
        assert len(cfg.channels) == len(cfg.down)
        layers = [conv3x3(cfg.img_channels, cfg.channels[0])]
        for i in range(len(cfg.channels)):
            layers.append(SmallResBlock(cfg.channels[max(0, i - 1)], cfg.channels[i]))
            if cfg.down[i]:
                layers.append(nn.MaxPool2d(2))
        self.encoder = nn.Sequential(*layers)


class ActorCritic(NativeStateMixin, nn.Module):
    _NATIVE_PREFIX = "dmd_actor_critic_"
    _WS_POOL_CAP = 64   # one workspace per live autograd node of the imagined rollout (15 steps + burn-in calls)

    def __init__(self, cfg: ActorCriticConfig) -> None:
        super().__init__()
        self.cfg = cfg
        self.encoder = ActorCriticEncoder(cfg)
        self.lstm_dim = cfg.lstm_dim
        input_dim_lstm = cfg.channels[-1] * (cfg.img_size // 2 ** (sum(cfg.down))) ** 2
        self.lstm = nn.LSTMCell(input_dim_lstm, cfg.lstm_dim)
        self.critic_linear = nn.Linear(cfg.lstm_dim, 1)
        self.actor_linear = nn.Linear(cfg.lstm_dim, cfg.num_actions)
        for lin in (self.actor_linear, self.critic_linear):  # actor_critic.py:50-53
            lin.weight.data.fill_(0)
            lin.bias.data.fill_(0)
        init_lstm(self.lstm)
        self.env_loop = None
        self.loss_cfg = None
        # True: the nodes of a backward pass accumulate their parameter gradients natively and `.grad` is set when the pass ends
        # (what `loss.backward()` needs).  False: every node returns its gradients to autograd (needed for torch.autograd.grad).
        self.accumulate_native_grads = True

    @property
    def device(self) -> torch.device:  # actor_critic.py:59-61
        return self.lstm.weight_hh.device

    def setup_training(self, rl_env, loss_cfg: ActorCriticLossConfig) -> None:  # actor_critic.py:63-66
        assert self.env_loop is None and self.loss_cfg is None
        self.env_loop = make_env_loop(rl_env, self)
        self.loss_cfg = loss_cfg

    # ------------------------------------------------------------------ native plumbing
    def _native_config(self):
        c = self.cfg
        cc = _lib.ActorCriticConfigC()
        cc.lstm_dim, cc.img_channels, cc.img_size, cc.num_levels = c.lstm_dim, c.img_channels, c.img_size, len(c.channels)
        for i in range(len(c.channels)):
            cc.channels[i], cc.down[i] = int(c.channels[i]), int(bool(c.down[i]))
        cc.num_actions = int(c.num_actions)
        return cc

    def _native_forward(self, obs: Tensor, hx: Tensor, cx: Tensor, ws: Tensor):
        lib = _lib.lib()
        h = self._native()
        b = obs.size(0)
        logits = torch.empty(b, self.cfg.num_actions, device=obs.device)
        val = torch.empty(b, device=obs.device)
        hx_o, cx_o = torch.empty_like(hx), torch.empty_like(cx)
        _lib.check(lib.dmd_actor_critic_forward(h, b, obs.data_ptr(), hx.data_ptr(), cx.data_ptr(), logits.data_ptr(),
                                                val.data_ptr(), hx_o.data_ptr(), cx_o.data_ptr(), ws.data_ptr(), ws.numel(),
                                                _lib.current_stream()))
        return logits, val, hx_o, cx_o

    # ------------------------------------------------------------------ reference surface
    def predict_act_value(self, obs: Tensor, hx_cx: Tuple[Tensor, Tensor]) -> ActorCriticOutput:  # actor_critic.py:68-73
        assert obs.ndim == 4
        lib = _lib.lib()
        h = self._native()
        hx, cx = hx_cx
        obs_, hx_, cx_ = obs.float().contiguous(), hx.float().contiguous(), cx.float().contiguous()
        need = lib.dmd_actor_critic_workspace_bytes(h, obs.size(0))
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # one autograd node per call: the imagined rollout back-propagates through time across these nodes
            params = [p for p in self.parameters()]
            logits, val, hx_o, cx_o = _PredictActValueFn.apply(self, obs_, hx_, cx_, *params)
            return ActorCriticOutput(logits, val, (hx_o, cx_o))
        if self._ws is None or self._ws.numel() < need or self._ws.device != obs.device:
            self._ws = torch.empty(need, dtype=torch.uint8, device=obs.device)
        logits, val, hx_o, cx_o = self._native_forward(obs_, hx_, cx_, self._ws)
        return ActorCriticOutput(logits, val, (hx_o, cx_o))

    def forward(self) -> LossAndLogs:  # actor_critic.py:75-98
        """REINFORCE with a lambda-return baseline over one imagined rollout of `backup_every` steps."""
        cfg = self.loss_cfg
        self.__dict__.pop("_grad_acc", None)   # a backward pass that died half-way must not leak into this update
        _, act, rew, end, trunc, logits, val, val_bootstrap, _ = self.env_loop.send(cfg.backup_every)
        policy = Categorical(logits=logits, validate_args=False)
        entropy = policy.entropy().mean()
        target = compute_lambda_returns(rew, end, trunc, val_bootstrap, cfg.gamma, cfg.lambda_)
        advantage = (target - val).detach()
        loss_actions = (-policy.log_prob(act) * advantage).mean()
        loss_values = cfg.weight_value_loss * F.mse_loss(val, target)
        loss_entropy = -cfg.weight_entropy_loss * entropy
        loss = loss_actions + loss_entropy + loss_values
        logs = {
            "policy_entropy": entropy.detach() / math.log(2),
            "loss_actions": loss_actions.detach(),
            "loss_entropy": loss_entropy.detach(),
            "loss_values": loss_values.detach(),
            "loss_total": loss.detach(),
        }
        return loss, logs


@torch.no_grad()
def compute_lambda_returns(rew: Tensor, end: Tensor, trunc: Tensor, val_bootstrap: Tensor, gamma: float, lambda_: float) -> Tensor:
    """Lambda-returns with sign-clipped rewards, episode ends and truncations (actor_critic.py:116-143).  CUDA inputs run in
    one native kernel (one thread per environment walking time backwards, fp32 operations in the reference's order:
    bit-identical); CPU inputs (host-logic tests only) evaluate the same recursion with torch ops."""
    assert rew.ndim == 2 and rew.size() == end.size() == trunc.size() == val_bootstrap.size()
    if rew.is_cuda:
        b, t = rew.shape
        out = torch.empty(b, t, dtype=torch.float32, device=rew.device)
        _lib.check(_lib.lib().dmd_lambda_returns(rew.float().contiguous().data_ptr(), end.long().contiguous().data_ptr(),
                                                 trunc.long().contiguous().data_ptr(), val_bootstrap.float().contiguous().data_ptr(),
                                                 out.data_ptr(), b, t, float(gamma), float(lambda_), _lib.current_stream()))
        return out
    stop = (end + trunc).clip(max=1)
    out = rew.sign() + (1 - end) * gamma * ((1 - trunc) * (1 - lambda_) + trunc) * val_bootstrap
    if lambda_ == 0:
        return out
    carry = val_bootstrap[:, -1]
    for t in range(rew.size(1) - 1, -1, -1):
        out[:, t] += stop[:, t].logical_not() * gamma * lambda_ * carry
        carry = out[:, t]
    return out


class _PredictActValueFn(torch.autograd.Function):
    """predict_act_value as one autograd node: forward = dmd_actor_critic_forward into a workspace that is kept until
    backward = dmd_actor_critic_backward (gradients wrt hx, cx and every parameter; obs needs none)."""

    @staticmethod
    def forward(ctx, module, obs, hx, cx, *params):
        lib = _lib.lib()
        h = module._native()
        ws = module._acquire_ws(lib.dmd_actor_critic_workspace_bytes(h, obs.size(0)))
        logits, val, hx_o, cx_o = module._native_forward(obs, hx.detach(), cx.detach(), ws)
        ctx.module, ctx.ws, ctx.b = module, ws, obs.size(0)
        ctx.under_ddp = module._under_ddp()
        ctx.save_for_backward(hx.detach(), cx.detach(), hx_o)
        ctx.set_materialize_grads(False)
        return logits, val, hx_o, cx_o

    @staticmethod
    def backward(ctx, g_logits, g_val, g_hx, g_cx):
        lib = _lib.lib()
        module = ctx.module
        h = module._native()
        hx, cx, hx_o = ctx.saved_tensors
        dev = hx.device
        offs, nums, total = module._grad_views_layout()
        g_hx_in, g_cx_in = torch.empty_like(hx), torch.empty_like(cx)
        need = lib.dmd_actor_critic_backward_scratch_bytes(h, ctx.b)
        scratch = module.__dict__.get("_bwd_scratch")
        if scratch is None or scratch.numel() < need or scratch.device != dev:
            scratch = module.__dict__["_bwd_scratch"] = torch.empty(need, dtype=torch.uint8, device=dev)

        def c(t):
            return None if t is None else t.float().contiguous()

        gl, gv, gh, gc = c(g_logits), c(g_val), c(g_hx), c(g_cx)
        args = (h, ctx.b, hx.data_ptr(), cx.data_ptr(), hx_o.data_ptr(), _lib.ptr(gl), _lib.ptr(gv), _lib.ptr(gh), _lib.ptr(gc))
        tail = (g_hx_in.data_ptr(), g_cx_in.data_ptr(), ctx.ws.data_ptr(), scratch.data_ptr(), scratch.numel(), _lib.current_stream())
        if module.accumulate_native_grads:
            # One flat gradient buffer per backward pass: every node of the BPTT graph ADDS into it natively, and a callback that the
            # autograd engine runs once the pass is complete hands it to the parameters.  (Returning ~40 gradient views per node
            # instead makes autograd's AccumulateGrad launch ~40 tiny additions for each of the ~60 nodes of a rollout.)  Under DDP
            # one node hands autograd views of the buffer instead (NativeStateMixin._pass_param_grads).
            flat = module.__dict__.get("_grad_acc")
            if flat is None:
                flat = module.__dict__["_grad_acc"] = torch.empty(total, dtype=torch.float32, device=dev)
                _lib.check(lib.dmd_actor_critic_backward(*args, flat.data_ptr(), total, *tail))
                torch.autograd.Variable._execution_engine.queue_callback(module._adopt_accumulated_grads)
            else:
                _lib.check(lib.dmd_actor_critic_backward_accumulate(*args, flat.data_ptr(), total, *tail))
            module._release_ws(ctx.ws, module._WS_POOL_CAP)
            return (None, None, g_hx_in, g_cx_in, *module._pass_param_grads(ctx, flat))
        flat = torch.empty(total, dtype=torch.float32, device=dev)
        _lib.check(lib.dmd_actor_critic_backward(*args, flat.data_ptr(), total, *tail))
        module._release_ws(ctx.ws, module._WS_POOL_CAP)
        grads = [flat[o:o + n].view_as(p) for (o, n), p in zip(zip(offs, nums), module.parameters())]
        return (None, None, g_hx_in, g_cx_in, *grads)
