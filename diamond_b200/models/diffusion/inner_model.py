"""InnerModel (reference: src/models/diffusion/inner_model.py) bound to the native denoiser executor.  `obs` is an fp32
frame stack (B, T*C, H, W), or a `frames.U8FrameStack` whose table already holds obs / sigma_data."""
import ctypes as C
from dataclasses import dataclass
from typing import List, Optional

import torch
from torch import Tensor
import torch.nn as nn

from ... import _lib
from ...frames import U8FrameStack
from ...utils import NativeStateMixin
from ..blocks import FourierFeatures, GroupNorm, UNet, conv3x3


@dataclass
class InnerModelConfig:  # inner_model.py:13-21
    img_channels: int
    num_steps_conditioning: int
    cond_channels: int
    depths: List[int]
    channels: List[int]
    attn_depths: List[bool]
    num_actions: Optional[int] = None


class InnerModel(NativeStateMixin, nn.Module):
    _NATIVE_PREFIX = "dmd_denoiser_"
    # A training workspace holds one forward's activations until its backward has run; an autoregressive Denoiser.forward
    # therefore holds several at once
    _WS_POOL_CAP = 4

    def __init__(self, cfg: InnerModelConfig) -> None:  # inner_model.py:24-42 (same registration order)
        super().__init__()
        self.cfg = cfg
        self.noise_emb = FourierFeatures(cfg.cond_channels)
        self.act_emb = nn.Sequential(
            nn.Embedding(cfg.num_actions, cfg.cond_channels // cfg.num_steps_conditioning),
            nn.Flatten(),
        )
        self.cond_proj = nn.Sequential(
            nn.Linear(cfg.cond_channels, cfg.cond_channels),
            nn.SiLU(),
            nn.Linear(cfg.cond_channels, cfg.cond_channels),
        )
        self.conv_in = conv3x3((cfg.num_steps_conditioning + 1) * cfg.img_channels, cfg.channels[0])
        self.unet = UNet(cfg.cond_channels, cfg.depths, cfg.channels, cfg.attn_depths)
        self.norm_out = GroupNorm(cfg.channels[0])
        self.conv_out = conv3x3(cfg.channels[0], cfg.img_channels)
        nn.init.zeros_(self.conv_out.weight)

    # ------------------------------------------------------------------ native executor plumbing
    @property
    def device(self) -> torch.device:
        return self.noise_emb.weight.device

    def _native_config(self, sigma_data: float, sigma_offset_noise: float):
        c = self.cfg
        cc = _lib.DenoiserConfigC()
        cc.img_channels, cc.num_steps_conditioning, cc.cond_channels = c.img_channels, c.num_steps_conditioning, c.cond_channels
        cc.num_levels = len(c.channels)
        for i in range(len(c.channels)):
            cc.depths[i], cc.channels[i], cc.attn_depths[i] = int(c.depths[i]), int(c.channels[i]), int(bool(c.attn_depths[i]))
        cc.num_actions = int(c.num_actions)
        cc.sigma_data, cc.sigma_offset_noise = sigma_data, sigma_offset_noise
        return cc

    def native(self, sigma_data: float = 0.5, sigma_offset_noise: float = 0.3):
        """Returns the native handle with up-to-date weights (re-packs when any parameter changed)."""
        return self._native_handle(float(sigma_data), float(sigma_offset_noise))

    def _native(self):
        return self.native()

    def workspace(self, nbytes: int) -> Tensor:
        dev = self.device
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        return self._ws

    def check_frame_stack(self, obs: U8FrameStack, b: int, h: int, w: int) -> None:
        want = (b, self.cfg.num_steps_conditioning, self.cfg.img_channels, h, w)
        if tuple(obs.shape) != want:
            raise ValueError(f"InnerModel: uint8 frame stack of shape {tuple(obs.shape)}, expected {want}")

    # ------------------------------------------------------------------ reference surface
    def forward(self, noisy_next_obs: Tensor, c_noise: Tensor, obs: Tensor, act: Tensor) -> Tensor:  # inner_model.py:44-49
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # training: native forward that keeps its activations + native backward, behind one autograd node whose inputs
            # are the leaf parameters (so .grad lands where configure_opt / DDP expect it, utils.py:105-106,129-166)
            return _InnerModelFn.apply(self, noisy_next_obs, c_noise, obs, act, *self.parameters())
        lib = _lib.lib()
        h = self.native()
        b, _, hh, ww = noisy_next_obs.shape
        noisy = noisy_next_obs.float().contiguous()
        cn = c_noise.float().contiguous().reshape(-1)
        act_ = act.long().contiguous()
        out = torch.empty_like(noisy)
        need = lib.dmd_denoiser_workspace_bytes(h, b, hh, ww)
        ws = self.workspace(need)
        if isinstance(obs, U8FrameStack):
            self.check_frame_stack(obs, b, hh, ww)
            _lib.check(lib.dmd_inner_model_forward_u8(h, b, hh, ww, noisy.data_ptr(), cn.data_ptr(), int(cn.numel() == 1),
                                                      C.byref(obs.c_struct()), act_.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                                      ws.numel(), _lib.current_stream()))
            return out
        obs_ = obs.float().contiguous()
        _lib.check(lib.dmd_inner_model_forward(h, b, hh, ww, noisy.data_ptr(), cn.data_ptr(), int(cn.numel() == 1),
                                               obs_.data_ptr(), act_.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                               _lib.current_stream()))
        return out


class _InnerModelFn(torch.autograd.Function):
    """InnerModel.forward under autograd: forward = dmd_inner_model_forward_train (activations stay in the training
    workspace), backward = dmd_denoiser_backward[_accumulate] (all parameter gradients in one flat buffer; see
    NativeStateMixin._native_param_grads for how it reaches `.grad`)."""

    @staticmethod
    def forward(ctx, module, noisy, c_noise, obs, act, *params):
        lib = _lib.lib()
        h = module.native()
        b, _, hh, ww = noisy.shape
        if isinstance(obs, U8FrameStack):
            module.check_frame_stack(obs, b, hh, ww)
        noisy_ = noisy.detach().float().contiguous()
        cn = c_noise.detach().float().contiguous().reshape(-1)
        act_ = act.long().contiguous()
        out = torch.empty_like(noisy_)
        ws = module._acquire_ws(lib.dmd_denoiser_train_workspace_bytes(h, b, hh, ww))
        if isinstance(obs, U8FrameStack):   # uint8 frame stack, read in place (its tensors are kept like obs_)
            obs_ = obs
            _lib.check(lib.dmd_inner_model_forward_train_u8(h, b, hh, ww, noisy_.data_ptr(), cn.data_ptr(), int(cn.numel() == 1),
                                                            C.byref(obs.c_struct()), act_.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                                            ws.numel(), _lib.current_stream()))
        else:
            obs_ = obs.detach().float().contiguous()
            _lib.check(lib.dmd_inner_model_forward_train(h, b, hh, ww, noisy_.data_ptr(), cn.data_ptr(), int(cn.numel() == 1),
                                                         obs_.data_ptr(), act_.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                         _lib.current_stream()))
        ctx.module, ctx.shape, ctx.ws, ctx.keep = module, (b, hh, ww), ws, (noisy_, obs_, cn, act_)
        ctx.under_ddp = module._under_ddp()
        return out

    @staticmethod
    def backward(ctx, grad_out):
        lib = _lib.lib()
        module = ctx.module
        h = module.native()
        b, hh, ww = ctx.shape
        g = grad_out.float().contiguous()

        def run(flat, accumulate):
            fn = lib.dmd_denoiser_backward_accumulate if accumulate else lib.dmd_denoiser_backward
            _lib.check(fn(h, b, hh, ww, g.data_ptr(), flat.data_ptr(), flat.numel(), ctx.ws.data_ptr(), _lib.current_stream()))
        grads = module._native_param_grads(ctx, run)
        module._release_ws(ctx.ws, module._WS_POOL_CAP)
        return (None, None, None, None, None, *grads)
