"""RewEndModel (reference: src/models/rew_end_model.py) with native sm_90a inference and training (SURVEY.md 8 f1, f2).

The reward / termination model runs once per imagined step between the sampler and the policy (world_model_env.py:97) and
over the burn-in frames of every fresh episode (:120-129).  Parameters live under the reference's names (state_dict keys,
`Agent.load`, `configure_opt`'s isinstance split keep working); the arithmetic — encoder ResBlocks at C = 32 with FiLM on
the action embedding, two attention blocks, LSTM over time, SiLU head — runs in `dmd_rew_end_predict`.
Training (`forward`, rew_end_model.py:57-90) keeps the reference's host logic and loss in torch; with gradients enabled,
`predict_rew_end` is one autograd node whose forward is `dmd_rew_end_forward_train` and whose backward is
`dmd_rew_end_backward` (BPTT through the LSTM, the encoder on the denoiser's backward plan).
uint8 frames (Episode.save's levels) go through the `_u8` entry points, with one kind per frame (frames.py): obs / next_obs
are then uint8 (b, t, C, S, S) and `kinds` = (obs kinds, next_obs kinds), each (b, t) uint8."""
import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from torch.autograd.function import once_differentiable

from .. import _lib, torch_ops
from .. import frames as frames_u8
from ..utils import NativeStateMixin, init_lstm
from .blocks import Downsample, ResBlocks, _NativeOnly, conv3x3


@dataclass
class RewEndModelConfig:  # rew_end_model.py:15-24
    lstm_dim: int
    img_channels: int
    img_size: int
    cond_channels: int
    depths: List[int]
    channels: List[int]
    attn_depths: List[int]
    num_actions: Optional[int] = None


class RewEndEncoder(_NativeOnly):  # rew_end_model.py:93-125 (parameter container; executed natively)
    def __init__(self, in_channels: int, cond_channels: int, depths: List[int], channels: List[int], attn_depths: List[int]) -> None:
        super().__init__()
        assert len(depths) == len(channels) == len(attn_depths)
        self.conv_in = conv3x3(in_channels, channels[0])
        blocks = []
        for i, n in enumerate(depths):
            c1, c2 = channels[max(0, i - 1)], channels[i]
            blocks.append(ResBlocks([c1] + [c2] * (n - 1), [c2] * n, cond_channels, attn_depths[i]))
        blocks.append(ResBlocks([channels[-1]] * 2, [channels[-1]] * 2, cond_channels, True))
        self.blocks = nn.ModuleList(blocks)
        self.downsamples = nn.ModuleList([nn.Identity()] + [Downsample(c) for c in channels[:-1]] + [nn.Identity()])


class RewEndModel(NativeStateMixin, nn.Module):
    _NATIVE_PREFIX = "dmd_rew_end_"

    def __init__(self, cfg: RewEndModelConfig) -> None:  # rew_end_model.py:27-41 (same registration order)
        super().__init__()
        self.cfg = cfg
        self.encoder = RewEndEncoder(2 * cfg.img_channels, cfg.cond_channels, cfg.depths, cfg.channels, cfg.attn_depths)
        self.act_emb = nn.Embedding(cfg.num_actions, cfg.cond_channels)
        input_dim_lstm = cfg.channels[-1] * (cfg.img_size // 2 ** (len(cfg.depths) - 1)) ** 2
        self.lstm = nn.LSTM(input_dim_lstm, cfg.lstm_dim, batch_first=True)
        self.head = nn.Sequential(nn.Linear(cfg.lstm_dim, cfg.lstm_dim), nn.SiLU(), nn.Linear(cfg.lstm_dim, 3 + 2, bias=False))
        init_lstm(self.lstm)

    @property
    def device(self) -> torch.device:
        return self.act_emb.weight.device

    def _native_config(self):
        c = self.cfg
        cc = _lib.RewEndConfigC()
        cc.lstm_dim, cc.img_channels, cc.img_size, cc.cond_channels, cc.num_levels = c.lstm_dim, c.img_channels, c.img_size, c.cond_channels, len(c.channels)
        for i in range(len(c.channels)):
            cc.depths[i], cc.channels[i], cc.attn_depths[i] = int(c.depths[i]), int(c.channels[i]), int(bool(c.attn_depths[i]))
        cc.num_actions = int(c.num_actions)
        return cc

    # a training workspace holds one forward's activations until its backward has run
    _WS_POOL_CAP = 2
    _ws_bytes = None   # rows, deterministic -> inference workspace size

    def predict_rew_end(self, obs: Tensor, act: Tensor, next_obs: Tensor, hx_cx: Optional[Tuple[Tensor, Tensor]] = None,
                        kinds: Optional[Tuple[Tensor, Tensor]] = None) -> Tuple[Tensor, Tensor, Tuple[Tensor, Tensor]]:
        # rew_end_model.py:42-55.  hx_cx: each (1, b, lstm_dim) like torch.nn.LSTM
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            b = obs.size(0)
            hx = cx = None
            if hx_cx is not None:
                hx, cx = hx_cx[0].reshape(b, -1), hx_cx[1].reshape(b, -1)
            src = self._u8_sources(obs, next_obs, kinds)
            rew, end, hx_o, cx_o = _RewEndFn.apply(self, obs, act, next_obs, hx, cx, src, *self.parameters())
            return rew, end, (hx_o.unsqueeze(0), cx_o.unsqueeze(0))
        return self._predict(obs, act, next_obs, hx_cx, kinds)

    def _u8_sources(self, obs: Tensor, next_obs: Tensor, kinds: Optional[Tuple[Tensor, Tensor]]):
        """None for fp32 frames; for uint8 frames the two U8FrameStacks the `_u8` entry points read (one decode table)."""
        if obs.dtype != torch.uint8 and next_obs.dtype != torch.uint8:
            return None
        if obs.dtype != next_obs.dtype or kinds is None:
            raise ValueError("RewEndModel: uint8 obs and next_obs go together, with kinds = (obs kinds, next_obs kinds)")
        want = (obs.size(0), obs.size(1), self.cfg.img_channels, self.cfg.img_size, self.cfg.img_size)
        if tuple(obs.shape) != want or tuple(next_obs.shape) != want:
            raise ValueError(f"RewEndModel: uint8 obs / next_obs of shapes {tuple(obs.shape)} / {tuple(next_obs.shape)}, expected {want}")
        table = frames_u8.decode_table(obs.device)
        return frames_u8.U8FrameStack(obs, kinds[0], table), frames_u8.U8FrameStack(next_obs, kinds[1], table)

    @torch.no_grad()
    def _predict(self, obs: Tensor, act: Tensor, next_obs: Tensor, hx_cx: Optional[Tuple[Tensor, Tensor]] = None,
                 kinds: Optional[Tuple[Tensor, Tensor]] = None) -> Tuple[Tensor, Tensor, Tuple[Tensor, Tensor]]:
        b, t = obs.shape[:2]
        src = self._u8_sources(obs, next_obs, kinds)
        act_ = act.long().contiguous()
        hx = cx = None
        if hx_cx is not None:
            hx, cx = hx_cx[0].reshape(b, -1).float().contiguous(), hx_cx[1].reshape(b, -1).float().contiguous()
        ws = self.predict_workspace(b * t)
        if src is not None:
            lib = _lib.lib()
            h = self._native()
            rew, end, hx_o, cx_o = self._new_outputs(b, t, obs.device)
            _lib.check(lib.dmd_rew_end_predict_u8(h, b, t, C.byref(src[0].c_struct()), C.byref(src[1].c_struct()), act_.data_ptr(),
                                                  _lib.ptr(hx), _lib.ptr(cx), rew.data_ptr(), end.data_ptr(), hx_o.data_ptr(),
                                                  cx_o.data_ptr(), ws.data_ptr(), ws.numel(), _lib.current_stream()))
            return rew, end, (hx_o.unsqueeze(0), cx_o.unsqueeze(0))
        # one diamond_b200::rew_end_predict op, so that torch.compile traces it whole
        rew, end, hx_o, cx_o = torch_ops.rew_end_predict(torch_ops.key_of(self), obs.float().contiguous(), act_,
                                                         next_obs.float().contiguous(), hx, cx, ws, self._state_tensors())
        return rew, end, (hx_o.unsqueeze(0), cx_o.unsqueeze(0))

    def _new_outputs(self, b: int, t: int, dev):
        d = self.cfg.lstm_dim
        return (torch.empty(b, t, 3, device=dev), torch.empty(b, t, 2, device=dev), torch.empty(b, d, device=dev),
                torch.empty(b, d, device=dev))

    def _predict_native(self, obs: Tensor, act: Tensor, next_obs: Tensor, hx: Optional[Tensor], cx: Optional[Tensor], ws: Tensor):
        """dmd_rew_end_predict on fp32 frames (the body of the diamond_b200::rew_end_predict op)."""
        lib = _lib.lib()
        h = self._native()
        b, t = obs.shape[:2]
        rew, end, hx_o, cx_o = self._new_outputs(b, t, obs.device)
        _lib.check(lib.dmd_rew_end_predict(h, b, t, obs.data_ptr(), next_obs.data_ptr(), act.data_ptr(), _lib.ptr(hx), _lib.ptr(cx),
                                           rew.data_ptr(), end.data_ptr(), hx_o.data_ptr(), cx_o.data_ptr(), ws.data_ptr(),
                                           ws.numel(), _lib.current_stream()))
        return rew, end, hx_o, cx_o

    def predict_workspace(self, rows: int) -> Tensor:
        """The inference workspace for `rows` = b * t frames.  Its size is asked of the native layer once per row count and
        mode, so that a compiled caller traces this as plain attribute reads (WorldModelEnv.reset sees its shape first)."""
        key = (rows, torch.are_deterministic_algorithms_enabled())
        sizes = self._ws_bytes
        if sizes is None:
            sizes = self._ws_bytes = {}
        if key not in sizes:
            need = _lib.lib().dmd_rew_end_workspace_bytes(self._native(), rows)
            if need == 0:
                raise RuntimeError("diamond_b200: " + _lib.lib().dmd_last_error().decode())
            sizes[key] = need
        dev = self.device
        if self._ws is None or self._ws.numel() < sizes[key] or self._ws.device != dev:
            self._ws = torch.empty(sizes[key], dtype=torch.uint8, device=dev)
        return self._ws

    def forward(self, batch):  # rew_end_model.py:57-90
        obs = batch.obs[:, :-1]
        act = batch.act[:, :-1]
        next_obs = batch.obs[:, 1:]
        rew = batch.rew[:, :-1]
        end = batch.end[:, :-1]
        mask = batch.mask_padding[:, :-1]

        # When dead, replace frame (gray padding) by true final obs; the write goes through the view into batch.obs
        dead = end.bool().any(dim=1)
        kinds = None
        if batch.obs.dtype == torch.uint8:
            # uint8 batch: one kind per frame; a float final observation is encoded (a frame off the level grid raises), a
            # uint8 one is taken as the bytes a real env decodes on the GPU (src/envs/env.py:89)
            all_kinds = frames_u8.kinds_from_mask(batch.mask_padding, batch.obs.shape[:2], batch.obs.device)
            if dead.any():
                finals = [i["final_observation"] for i, d in zip(batch.info, dead) if d]
                levels, fk = zip(*[(f, torch.tensor(frames_u8.KIND_GPU, dtype=torch.uint8, device=f.device))
                                   if f.dtype == torch.uint8 else frames_u8.encode(f) for f in finals])
                slot = end[dead].argmax(dim=1)
                next_obs[dead, slot] = torch.stack(levels).to(obs.device)
                all_kinds[:, 1:][dead, slot] = torch.stack([k.to(obs.device) for k in fk])
            kinds = (all_kinds[:, :-1], all_kinds[:, 1:])
        elif dead.any():
            final_obs = torch.stack([i["final_observation"] for i, d in zip(batch.info, dead) if d]).to(obs.device)
            next_obs[dead, end[dead].argmax(dim=1)] = final_obs

        logits_rew, logits_end, _ = self.predict_rew_end(obs, act, next_obs, **({} if kinds is None else {"kinds": kinds}))
        logits_rew = logits_rew[mask]
        logits_end = logits_end[mask]
        target_rew = rew[mask].sign().long().add(1)  # clipped to {-1, 0, 1}
        target_end = end[mask]

        loss_rew = F.cross_entropy(logits_rew, target_rew)
        loss_end = F.cross_entropy(logits_end, target_end)
        loss = loss_rew + loss_end

        metrics = {
            "loss_rew": loss_rew.detach(),
            "loss_end": loss_end.detach(),
            "loss_total": loss.detach(),
            "confusion_matrix": {
                "rew": confusion_matrix(logits_rew, target_rew, num_classes=3),
                "end": confusion_matrix(logits_end, target_end, num_classes=2),
            },
        }
        return loss, metrics


def confusion_matrix(logits: Tensor, target: Tensor, num_classes: int) -> Tensor:
    """torcheval.metrics.functional.multiclass_confusion_matrix for logits (N, num_classes): counts [true class, predicted
    class] (row = target, column = argmax), int64.  This follows torcheval's documented convention; it has not been compared
    with torcheval itself, which is not a dependency of this package."""
    n = num_classes
    return torch.bincount(target.long() * n + logits.detach().argmax(dim=1), minlength=n * n).view(n, n)


class _RewEndFn(torch.autograd.Function):
    """RewEndModel.predict_rew_end under autograd: forward = dmd_rew_end_forward_train (activations stay in the training
    workspace), backward = dmd_rew_end_backward[_accumulate] (all parameter gradients in one flat buffer, see
    NativeStateMixin._native_param_grads; the gradients wrt a carried (hx, cx) when the caller's state requires them)."""

    @staticmethod
    def forward(ctx, module, obs, act, next_obs, hx, cx, src, *params):
        lib = _lib.lib()
        h = module._native()
        b, t = obs.shape[:2]
        D = module.cfg.lstm_dim
        act_ = act.long().contiguous()
        hx_ = None if hx is None else hx.detach().float().contiguous()
        cx_ = None if cx is None else cx.detach().float().contiguous()
        f32 = dict(dtype=torch.float32, device=obs.device)
        rew = torch.empty(b, t, 3, **f32)
        end = torch.empty(b, t, 2, **f32)
        hx_o, cx_o = torch.empty(b, D, **f32), torch.empty(b, D, **f32)
        need = lib.dmd_rew_end_train_workspace_bytes(h, b, t)
        if need == 0:
            raise RuntimeError("diamond_b200: " + lib.dmd_last_error().decode())
        ws = module._acquire_ws(need)
        if src is not None:
            _lib.check(lib.dmd_rew_end_forward_train_u8(h, b, t, C.byref(src[0].c_struct()), C.byref(src[1].c_struct()), act_.data_ptr(),
                                                        _lib.ptr(hx_), _lib.ptr(cx_), rew.data_ptr(), end.data_ptr(), hx_o.data_ptr(),
                                                        cx_o.data_ptr(), ws.data_ptr(), ws.numel(), _lib.current_stream()))
        else:
            obs_, nxt_ = obs.detach().float().contiguous(), next_obs.detach().float().contiguous()
            _lib.check(lib.dmd_rew_end_forward_train(h, b, t, obs_.data_ptr(), nxt_.data_ptr(), act_.data_ptr(), _lib.ptr(hx_), _lib.ptr(cx_),
                                                     rew.data_ptr(), end.data_ptr(), hx_o.data_ptr(), cx_o.data_ptr(), ws.data_ptr(),
                                                     ws.numel(), _lib.current_stream()))
        ctx.module, ctx.shape, ctx.ws = module, (b, t), ws
        ctx.under_ddp = module._under_ddp()
        return rew, end, hx_o, cx_o

    @staticmethod
    @once_differentiable
    def backward(ctx, g_rew, g_end, g_hx, g_cx):
        lib = _lib.lib()
        module = ctx.module
        h = module._native()
        b, t = ctx.shape
        g_rew, g_end = g_rew.float().contiguous(), g_end.float().contiguous()
        g_hx = None if g_hx is None else g_hx.float().contiguous()
        g_cx = None if g_cx is None else g_cx.float().contiguous()
        g_hx_in = g_rew.new_empty(b, module.cfg.lstm_dim) if ctx.needs_input_grad[4] else None
        g_cx_in = g_rew.new_empty(b, module.cfg.lstm_dim) if ctx.needs_input_grad[5] else None

        def run(flat, accumulate):
            fn = lib.dmd_rew_end_backward_accumulate if accumulate else lib.dmd_rew_end_backward
            _lib.check(fn(h, b, t, g_rew.data_ptr(), g_end.data_ptr(), _lib.ptr(g_hx), _lib.ptr(g_cx), flat.data_ptr(), flat.numel(),
                          _lib.ptr(g_hx_in), _lib.ptr(g_cx_in), ctx.ws.data_ptr(), _lib.current_stream()))
        grads = module._native_param_grads(ctx, run)
        module._release_ws(ctx.ws, module._WS_POOL_CAP)
        return (None, None, None, None, g_hx_in, g_cx_in, None, *grads)
