"""DiffusionSampler (reference: src/models/diffusion/diffusion_sampler.py), whole loop in one native call."""
import ctypes as C
from dataclasses import dataclass
from typing import List, Tuple

import torch
from torch import Tensor

from ... import _lib, torch_ops
from .denoiser import Denoiser


@dataclass
class DiffusionSamplerConfig:  # diffusion_sampler.py:10-20
    num_steps_denoising: int
    sigma_min: float = 2e-3
    sigma_max: float = 5
    rho: int = 7
    order: int = 1
    s_churn: float = 0
    s_tmin: float = 0
    s_tmax: float = float("inf")
    s_noise: float = 1


def build_sigmas(num_steps: int, sigma_min: float, sigma_max: float, rho: int, device: torch.device) -> Tensor:
    # diffusion_sampler.py:61-66 (Karras et al. schedule), same fp32 torch expressions
    min_inv_rho = sigma_min ** (1 / rho)
    max_inv_rho = sigma_max ** (1 / rho)
    l = torch.linspace(0, 1, num_steps, device=device)
    sigmas = (max_inv_rho + l * (min_inv_rho - max_inv_rho)) ** rho
    return torch.cat((sigmas, sigmas.new_zeros(1)))


class DiffusionSampler:
    def __init__(self, denoiser: Denoiser, cfg: DiffusionSamplerConfig) -> None:
        self.denoiser = denoiser
        self.cfg = cfg
        # The schedule is host-known: computing it on CPU (bit-identical to the reference's CPU path) removes the two
        # device->host syncs per step the reference pays for `sigma <= ...` / `next_sigma == 0` (diffusion_sampler.py:39,47).
        self._sigmas_host = build_sigmas(cfg.num_steps_denoising, cfg.sigma_min, cfg.sigma_max, cfg.rho, torch.device("cpu"))
        self.sigmas = self._sigmas_host.to(denoiser.device)
        self.use_cuda_graph = True
        self._n_sig = int(self._sigmas_host.numel())
        self._sig_arr = (C.c_float * self._n_sig)(*self._sigmas_host.tolist())
        self._sc = _lib.SamplerConfigC(self._n_sig, self._sig_arr, int(cfg.order), float(cfg.s_churn), float(cfg.s_tmin),
                                       float(min(cfg.s_tmax, 3.0e38)), 1.0)
        self._gamma = min(cfg.s_churn / (self._n_sig - 1), 2**0.5 - 1)
        self._ws_bytes = {}   # (b, h, w, deterministic) -> the denoiser's inference workspace size
        self._buf = {}   # persistent device buffers per (B, C, H, W): the native call (a CUDA graph) uses them in place

    def _buffers(self, b: int, t: int, c: int, h: int, w: int, device):
        key = (b, t, c, h, w, device)
        if key not in self._buf:
            self._buf = {key: dict(
                traj=torch.empty(self._n_sig, b, c, h, w, device=device),
                eps=torch.zeros(self._n_sig - 1, b, c, h, w, device=device) if self._gamma > 0 else None,
                obs=torch.empty(b, t * c, h, w, device=device), act=torch.empty(b, t, dtype=torch.long, device=device))}
        return self._buf[key]

    def _check_stack(self, t: int, c: int) -> None:
        # the reference fails inside act_emb / conv_in on a wrong stack depth (inner_model.py:45-46); fail as loudly here
        icfg = self.denoiser.cfg.inner_model
        if t != icfg.num_steps_conditioning or c != icfg.img_channels:
            raise RuntimeError(f"sample: frame stack of {t} x {c} channels, the denoiser is conditioned on "
                               f"{icfg.num_steps_conditioning} x {icfg.img_channels}")

    def _draw_noise(self, buf) -> None:
        """RNG stream parity with the reference: x first (diffusion_sampler.py:36), then one eps per churned step (:42)."""
        traj, eps = buf["traj"], buf["eps"]
        traj[0].copy_(torch.randn(*traj.shape[1:], device=traj.device))
        if eps is not None:
            for i, sigma in enumerate(self._sigmas_host[:-1].tolist()):
                if self.cfg.s_tmin <= sigma <= self.cfg.s_tmax:
                    eps[i].copy_(torch.randn(*traj.shape[1:], device=traj.device) * self.cfg.s_noise)

    def _workspace(self, b: int, h: int, w: int) -> Tensor:
        """The denoiser's inference workspace for (b, h, w).  Its size is asked of the native layer once per shape and mode, so
        that a compiled caller traces this as plain attribute reads (the shape is seen first by WorldModelEnv.reset)."""
        im = self.denoiser.inner_model
        key = (b, h, w, torch.are_deterministic_algorithms_enabled())
        sizes = self._ws_bytes
        if key not in sizes:
            den = self.denoiser
            sizes[key] = _lib.lib().dmd_denoiser_workspace_bytes(im.native(den.cfg.sigma_data, den.cfg.sigma_offset_noise), b, h, w)
        return im.workspace(sizes[key])

    def _sample_native(self, obs: Tensor, act: Tensor, ring_head: int, traj: Tensor, eps, out_x, ws: Tensor) -> None:
        lib = _lib.lib()
        den = self.denoiser
        hnd = den.inner_model.native(den.cfg.sigma_data, den.cfg.sigma_offset_noise)
        b, h, w = traj.shape[1], traj.shape[3], traj.shape[4]
        _lib.check(lib.dmd_sampler_sample(hnd, C.byref(self._sc), b, h, w, obs.data_ptr(), act.data_ptr(), ring_head,
                                          traj.data_ptr(), _lib.ptr(eps), _lib.ptr(out_x), ws.data_ptr(), ws.numel(),
                                          int(self.use_cuda_graph), _lib.current_stream()))

    @torch.no_grad()
    def sample(self, prev_obs: Tensor, prev_act: Tensor) -> Tuple[Tensor, List[Tensor]]:  # diffusion_sampler.py:31-58
        b, t, c, h, w = prev_obs.size()
        self._check_stack(t, c)
        buf = self._buffers(b, t, c, h, w, prev_obs.device)
        buf["obs"].copy_(prev_obs.reshape(b, t * c, h, w))   # stable addresses: the captured graph is replayed as is
        buf["act"].copy_(prev_act)
        self._draw_noise(buf)
        self._sample_native(buf["obs"], buf["act"], -1, buf["traj"], buf["eps"], None, self._workspace(b, h, w))
        traj = buf["traj"].clone()                           # the caller owns what it gets; the buffers are reused next call
        return traj[-1], list(traj.unbind(0))

    def prepare_ring(self, frames: Tensor) -> None:
        """Creates what sample_ring(frames, ...) keeps between calls -- its buffers, the native handle with packed weights and
        the workspace -- outside any compiled region, and marks the buffers static for the CUDA graphs of a compiled caller."""
        t, b, c, h, w = frames.size()
        self._check_stack(t, c)
        buf = self._buffers(b, t, c, h, w, frames.device)
        self._workspace(b, h, w)
        torch_ops.key_of(self)
        torch_ops.mark_static(buf["traj"], buf["eps"])

    @torch.no_grad()
    def sample_ring(self, frames: Tensor, acts: Tensor, head: int) -> Tensor:
        """The WorldModelEnv path: `frames` (T, B, C, H, W) / `acts` (T, B) are the environment's resident ring buffers with
        logical slot k at physical slot (head + k) % T; the new frame is written straight into the ring slot `frames[head]`.
        Nothing is staged or rolled.  Returns the trajectory buffer (num_sigmas, B, C, H, W), valid until the next call.
        One `diamond_b200::sample_ring` op, so that torch.compile traces it whole."""
        t, b, c, h, w = frames.size()
        self._check_stack(t, c)
        buf = self._buffers(b, t, c, h, w, frames.device)
        self._draw_noise(buf)
        torch_ops.sample_ring(torch_ops.key_of(self), frames, acts, head, buf["traj"], buf["eps"], self._workspace(b, h, w),
                              self.denoiser.inner_model._state_tensors())
        return buf["traj"]
