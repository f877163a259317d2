"""InnerModel (reference: src/models/diffusion/inner_model.py) bound to the native denoiser executor."""
import ctypes as C
from dataclasses import dataclass
from typing import List, Optional

import torch
from torch import Tensor
import torch.nn as nn

from ... import _lib
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
        # native state (not part of state_dict)
        self._h = None
        self._h_key = None
        self._packed = None
        self._wkey = None
        self._ws = None

    # ------------------------------------------------------------------ native executor plumbing
    def __del__(self):
        try:
            if self._h is not None:
                _lib.lib().dmd_denoiser_destroy(self._h)
        except Exception:
            pass

    def native(self, sigma_data: float = 0.5, sigma_offset_noise: float = 0.3):
        """Returns the native handle with up-to-date weights (re-packs when any parameter changed)."""
        lib = _lib.lib()
        dev = self.noise_emb.weight.device
        if dev.type != "cuda":
            raise RuntimeError("diamond_b200 runs on CUDA (sm_90a) only; move the model to a cuda device")
        self.require_current_device(dev)
        key = (float(sigma_data), float(sigma_offset_noise), dev.index)
        if self._h is None or self._h_key != key:
            if self._h is not None:
                lib.dmd_denoiser_destroy(self._h)
            c = self.cfg
            cc = _lib.DenoiserConfigC()
            cc.img_channels, cc.num_steps_conditioning, cc.cond_channels = c.img_channels, c.num_steps_conditioning, c.cond_channels
            cc.num_levels = len(c.channels)
            for i in range(len(c.channels)):
                cc.depths[i], cc.channels[i], cc.attn_depths[i] = int(c.depths[i]), int(c.channels[i]), int(bool(c.attn_depths[i]))
            cc.num_actions = int(c.num_actions)
            cc.sigma_data, cc.sigma_offset_noise = float(sigma_data), float(sigma_offset_noise)
            h = lib.dmd_denoiser_create(C.byref(cc))
            if not h:
                raise RuntimeError("diamond_b200: " + lib.dmd_last_error().decode())
            self._h, self._h_key, self._wkey, self._packed = h, key, None, None
        tensors = self._state_tensors()
        wkey = tuple((t.data_ptr(), t._version) for t in tensors)
        if wkey != self._wkey:
            n = lib.dmd_denoiser_num_tensors(self._h)
            if n != len(tensors):
                raise RuntimeError(f"native denoiser expects {n} tensors, module has {len(tensors)}")
            for t in tensors:
                if t.dtype != torch.float32 or not t.is_contiguous():
                    raise RuntimeError("parameters must be contiguous fp32")
            if self._packed is None:
                self._packed = torch.empty(lib.dmd_denoiser_packed_bytes(self._h), dtype=torch.uint8, device=dev)
            arr = (C.c_void_p * n)(*[t.data_ptr() for t in tensors])
            _lib.check(lib.dmd_denoiser_set_weights(self._h, arr, n, self._packed.data_ptr(), _lib.current_stream()))
            self._wkey = wkey
        return self._h

    def workspace(self, nbytes: int) -> Tensor:
        dev = self.noise_emb.weight.device
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        return self._ws

    # ------------------------------------------------------------------ training plumbing
    def grad_layout(self):
        """(offsets, numels, total) of the flat fp32 gradient buffer the native backward fills (state_dict order)."""
        lib = _lib.lib()
        h = self.native()
        n = lib.dmd_denoiser_num_tensors(h)
        offs, nums = (C.c_longlong * n)(), (C.c_longlong * n)()
        total = lib.dmd_denoiser_grad_layout(h, offs, nums, n)
        if total < 0:
            raise RuntimeError("diamond_b200: " + lib.dmd_last_error().decode())
        return list(offs), list(nums), int(total)

    def acquire_train_workspace(self, nbytes: int) -> Tensor:
        """A training workspace holds one forward's activations until its backward has run; an autoregressive
        Denoiser.forward therefore holds several at once.  Buffers are pooled and reused across optimizer steps."""
        dev = self.noise_emb.weight.device
        pool = self.__dict__.setdefault("_tws_pool", [])
        for i, ws in enumerate(pool):
            if ws.numel() >= nbytes and ws.device == dev:
                return pool.pop(i)
        return torch.empty(nbytes, dtype=torch.uint8, device=dev)

    def release_train_workspace(self, ws: Tensor) -> None:
        pool = self.__dict__.setdefault("_tws_pool", [])
        if len(pool) < 4:
            pool.append(ws)

    # ------------------------------------------------------------------ reference surface
    def forward(self, noisy_next_obs: Tensor, c_noise: Tensor, obs: Tensor, act: Tensor) -> Tensor:  # inner_model.py:44-49
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # training: native forward that keeps its activations + native backward, behind one autograd node whose inputs
            # are the leaf parameters (so .grad lands where configure_opt / DDP expect it, utils.py:105-106,129-166)
            names = [k for k, _ in self.named_parameters()]
            params = [p for _, p in self.named_parameters()]
            return _InnerModelFn.apply(self, names, noisy_next_obs, c_noise, obs, act, *params)
        lib = _lib.lib()
        h = self.native()
        b, _, hh, ww = noisy_next_obs.shape
        noisy, obs_ = noisy_next_obs.float().contiguous(), obs.float().contiguous()
        cn = c_noise.float().contiguous().reshape(-1)
        act_ = act.long().contiguous()
        out = torch.empty_like(noisy)
        need = lib.dmd_denoiser_workspace_bytes(h, b, hh, ww)
        ws = self.workspace(need)
        _lib.check(lib.dmd_inner_model_forward(h, b, hh, ww, noisy.data_ptr(), cn.data_ptr(), int(cn.numel() == 1),
                                               obs_.data_ptr(), act_.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                               _lib.current_stream()))
        return out


class _InnerModelFn(torch.autograd.Function):
    """InnerModel.forward under autograd: forward = dmd_inner_model_forward_train (activations stay in the training
    workspace), backward = dmd_denoiser_backward (all parameter gradients in one flat buffer, returned as views)."""

    @staticmethod
    def forward(ctx, module, names, noisy, c_noise, obs, act, *params):
        lib = _lib.lib()
        h = module.native()
        b, _, hh, ww = noisy.shape
        noisy_, obs_ = noisy.detach().float().contiguous(), obs.detach().float().contiguous()
        cn = c_noise.detach().float().contiguous().reshape(-1)
        act_ = act.long().contiguous()
        out = torch.empty_like(noisy_)
        ws = module.acquire_train_workspace(lib.dmd_denoiser_train_workspace_bytes(h, b, hh, ww))
        _lib.check(lib.dmd_inner_model_forward_train(h, b, hh, ww, noisy_.data_ptr(), cn.data_ptr(), int(cn.numel() == 1),
                                                     obs_.data_ptr(), act_.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                     _lib.current_stream()))
        ctx.module, ctx.names, ctx.shape, ctx.ws, ctx.keep = module, names, (b, hh, ww), ws, (noisy_, obs_, cn, act_)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        lib = _lib.lib()
        module = ctx.module
        h = module.native()
        b, hh, ww = ctx.shape
        offs, nums, total = module.grad_layout()
        flat = torch.empty(total, dtype=torch.float32, device=grad_out.device)
        g = grad_out.float().contiguous()
        _lib.check(lib.dmd_denoiser_backward(h, b, hh, ww, g.data_ptr(), flat.data_ptr(), total, ctx.ws.data_ptr(), _lib.current_stream()))
        index = {k: i for i, k in enumerate(module.state_dict().keys())}
        grads = []
        for name, p in zip(ctx.names, module.parameters()):
            i = index[name]
            grads.append(flat[offs[i]:offs[i] + nums[i]].view_as(p))
        module.release_train_workspace(ctx.ws)
        module.last_flat_grad = flat   # one contiguous buffer: what a data-parallel step all-reduces in a single collective
        return (None, None, None, None, None, None, *grads)
