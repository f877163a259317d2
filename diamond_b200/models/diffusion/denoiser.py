"""Denoiser: EDM preconditioning around the native InnerModel, with the reference's module surface
(src/models/diffusion/denoiser.py: same config schema, same public methods, same RNG draws in the same order).

How the work is split here:
* inference (`denoise`, and everything `DiffusionSampler` does) is ONE C-ABI call: the conditioners, the input packing, the
  U-Net, the wrap + truncating quantiser all run in the native executor (`dmd_denoiser_forward`, csrc/api.cu);
* training (`forward`) keeps the per-step scalar algebra of EDM on the host side in a small value object (`EdmCoefficients`,
  a handful of (B,)-sized torch ops) and runs the U-Net through the native autograd node of `InnerModel`;
* `compute_conditioners` / `compute_model_output` / `wrap_model_output` / `apply_noise` stay callable because the reference's
  callers and our parity tests use them; they are thin views over the same two mechanisms.
"""
from dataclasses import dataclass
from typing import Any, Dict, Optional, Tuple

import torch
from torch import Tensor
import torch.nn as nn

from ... import _lib
from ... import frames as frames_u8
from .inner_model import InnerModel, InnerModelConfig

LossAndLogs = Tuple[Tensor, Dict[str, Any]]


# ---------------------------------------------------------------------------------------------- hydra schema (config/agent)
@dataclass
class SigmaDistributionConfig:
    loc: float
    scale: float
    sigma_min: float
    sigma_max: float


@dataclass
class DenoiserConfig:
    inner_model: InnerModelConfig
    sigma_data: float
    sigma_offset_noise: float


@dataclass
class Conditioners:
    """What the reference hands around between its three compute_* steps (denoiser.py:18-23)."""
    c_in: Tensor
    c_out: Tensor
    c_skip: Tensor
    c_noise: Tensor


def add_dims(input: Tensor, n: int) -> Tensor:
    """Trailing singleton axes up to `n` dimensions (a per-sample scalar against an image batch)."""
    missing = n - input.ndim
    return input if missing <= 0 else input[(...,) + (None,) * missing]


class EdmCoefficients:
    """The four EDM preconditioning coefficients of a batch of noise levels, kept as flat (B,) fp32 vectors.

    Same expressions, in the same fp32 order, as denoiser.py:66-72 (and as `edm_conditioners` in csrc/aux_kernels.cuh, which
    the native inference path evaluates on the device):
        s      = sqrt(sigma^2 + offset^2)          total noise once the offset noise is accounted for
        c_in   = 1 / sqrt(s^2 + sd^2)              c_skip = sd^2 / (s^2 + sd^2)
        c_out  = s * sqrt(c_skip)                  c_noise = ln(s) / 4
    """

    __slots__ = ("c_in", "c_out", "c_skip", "c_noise")

    def __init__(self, sigma: Tensor, sigma_data: float, sigma_offset_noise: float) -> None:
        s = (sigma**2 + sigma_offset_noise**2).sqrt()
        total = s**2 + sigma_data**2
        self.c_in = 1 / total.sqrt()
        self.c_skip = sigma_data**2 / total
        self.c_out = s * self.c_skip.sqrt()
        self.c_noise = s.log() / 4

    def broadcast(self) -> Conditioners:
        """Image-shaped views: (B,1,1,1) for the three that scale frames, (B,) for the one that feeds the noise embedding."""
        return Conditioners(add_dims(self.c_in, 4), add_dims(self.c_out, 4), add_dims(self.c_skip, 4), add_dims(self.c_noise, 1))


def quantise_frame(x: Tensor) -> Tensor:
    """[-1, 1] -> the 256-level grid and back, TRUNCATING like a uint8 cast (denoiser.py:83); the native inference path does
    the same inside `wrap_update_kernel`."""
    levels = frames_u8.quantise_levels(x)
    return levels.div(255).mul(2).sub(1)


class _LogNormalSigma:
    """Noise-level distribution of training (denoiser.py:52-59): exp(N(loc, scale)) clipped to [sigma_min, sigma_max].
    One `torch.randn(n)` per call -- the RNG stream the fixtures replay."""

    def __init__(self, cfg: SigmaDistributionConfig) -> None:
        self.cfg = cfg

    def __call__(self, n: int, device: torch.device) -> Tensor:
        c = self.cfg
        return (torch.randn(n, device=device) * c.scale + c.loc).exp().clip(c.sigma_min, c.sigma_max)


class Denoiser(nn.Module):
    def __init__(self, cfg: DenoiserConfig) -> None:
        super().__init__()
        self.cfg = cfg
        self.inner_model = InnerModel(cfg.inner_model)
        self.sample_sigma_training: Optional[_LogNormalSigma] = None

    @property
    def device(self) -> torch.device:
        return self.inner_model.noise_emb.weight.device

    def setup_training(self, cfg: SigmaDistributionConfig) -> None:
        if self.sample_sigma_training is not None:
            raise AssertionError("setup_training was already called")   # the reference asserts (denoiser.py:53)
        self.sample_sigma_training = _LogNormalSigma(cfg)

    # ------------------------------------------------------------------ EDM pieces (reference surface)
    def _coefficients(self, sigma: Tensor) -> EdmCoefficients:
        return EdmCoefficients(sigma, self.cfg.sigma_data, self.cfg.sigma_offset_noise)

    def compute_conditioners(self, sigma: Tensor) -> Conditioners:
        return self._coefficients(sigma).broadcast()

    def apply_noise(self, x: Tensor, sigma: Tensor, sigma_offset_noise: float) -> Tensor:
        """x + per-(sample, channel) offset noise + sigma-scaled white noise; draws (b,c,1,1) then x-shaped, in that order."""
        offset = torch.randn(x.size(0), x.size(1), 1, 1, device=self.device) * sigma_offset_noise
        white = torch.randn_like(x)
        return x + offset + white * add_dims(sigma, x.ndim)

    def compute_model_output(self, noisy_next_obs: Tensor, obs: Tensor, act: Tensor, cs: Conditioners) -> Tensor:
        """F(c_in * x; c_noise, obs / sigma_data, act): InnerModel runs natively (with an autograd node when grad is enabled)."""
        return self.inner_model(noisy_next_obs * cs.c_in, cs.c_noise, obs / self.cfg.sigma_data, act)

    @torch.no_grad()
    def wrap_model_output(self, noisy_next_obs: Tensor, model_output: Tensor, cs: Conditioners) -> Tensor:
        return quantise_frame(cs.c_skip * noisy_next_obs + cs.c_out * model_output)

    # ------------------------------------------------------------------ inference: one native call
    def _native_forward(self, noisy: Tensor, sigma: Tensor, obs: Tensor, act: Tensor, want_model: bool, want_denoised: bool):
        """(model_output, denoised) of `dmd_denoiser_forward`; either may be skipped.  sigma: 1 or B elements."""
        lib = _lib.lib()
        im = self.inner_model
        handle = im.native(self.cfg.sigma_data, self.cfg.sigma_offset_noise)
        b, _, hh, ww = noisy.shape
        noisy_f, obs_f = noisy.float().contiguous(), obs.float().contiguous()
        sig = sigma.float().contiguous().reshape(-1).to(noisy.device)
        if sig.numel() not in (1, b):
            raise ValueError("sigma must have 1 or B elements")
        act_l = act.long().contiguous()
        model = torch.empty_like(noisy_f) if want_model else None
        denoised = torch.empty_like(noisy_f) if want_denoised else None
        ws = im.workspace(lib.dmd_denoiser_workspace_bytes(handle, b, hh, ww))
        _lib.check(lib.dmd_denoiser_forward(handle, b, hh, ww, noisy_f.data_ptr(), sig.data_ptr(), int(sig.numel() == 1),
                                            obs_f.data_ptr(), act_l.data_ptr(), _lib.ptr(model), _lib.ptr(denoised),
                                            ws.data_ptr(), ws.numel(), _lib.current_stream()))
        return model, denoised

    @torch.no_grad()
    def denoise(self, noisy_next_obs: Tensor, sigma: Tensor, obs: Tensor, act: Tensor) -> Tensor:
        return self._native_forward(noisy_next_obs, sigma, obs, act, want_model=False, want_denoised=True)[1]

    # ------------------------------------------------------------------ training
    def forward(self, batch) -> LossAndLogs:
        """Denoising loss over the autoregressive tail of a segment (denoiser.py:93-122).

        `batch.obs` is (B, T, C, H, W) with T = n_cond + steps.  Step i noises frame n_cond + i, predicts it from frames
        [i, n_cond + i) and their actions, and regresses the EDM target (x - c_skip * noisy) / c_out on the unpadded samples;
        the quantised prediction then REPLACES that frame, so later steps are conditioned on the model's own output.
        Random draws per step, in order: sigma, offset noise, white noise.

        A uint8 `batch.obs` (Episode.save's levels, padding where `batch.mask_padding` is False) computes the same loss and
        gradients as its fp32 decoding; see `_forward_u8`."""
        if self.sample_sigma_training is None:
            raise RuntimeError("call setup_training(SigmaDistributionConfig) first")
        if batch.obs.dtype == torch.uint8:
            return self._forward_u8(batch)
        n_cond = self.cfg.inner_model.num_steps_conditioning
        frames = batch.obs.clone()
        b, t_total, c, h, w = frames.shape
        steps = t_total - n_cond
        step_losses = []
        for i in range(steps):
            tgt = n_cond + i
            clean = frames[:, tgt]
            context = frames[:, i:tgt].reshape(b, n_cond * c, h, w)
            sigma = self.sample_sigma_training(b, self.device)
            noisy = self.apply_noise(clean, sigma, self.cfg.sigma_offset_noise)
            cs = self._coefficients(sigma).broadcast()
            out = self.compute_model_output(noisy, context, batch.act[:, i:tgt], cs)
            real = batch.mask_padding[:, tgt]
            regression_target = (clean - cs.c_skip * noisy) / cs.c_out
            step_losses.append(torch.nn.functional.mse_loss(out[real], regression_target[real]))
            frames[:, tgt] = self.wrap_model_output(noisy, out, cs)
        loss = sum(step_losses) / steps
        return loss, {"loss_denoising": loss.detach()}

    def _forward_u8(self, batch) -> LossAndLogs:
        """`forward` on a uint8 batch.  The working copy of the frames stays uint8, with one kind per frame (frames.py): the
        loaded frames decode as Episode.load does, padding as 0.0, and each write-back stores the quantiser's levels with
        the kind of a GPU decode.  Only the target frame is decoded in torch (for the noise and the regression target); the
        native pack kernel reads the context frames [i, n_cond + i) in place through the table of obs / sigma_data."""
        n_cond = self.cfg.inner_model.num_steps_conditioning
        frames = batch.obs.clone()
        b, t_total = frames.shape[:2]
        kinds = frames_u8.kinds_from_mask(batch.mask_padding, (b, t_total), frames.device)
        table = frames_u8.decode_table(frames.device)
        ctx_table = frames_u8.context_table(frames.device, self.cfg.sigma_data)
        steps = t_total - n_cond
        step_losses = []
        for i in range(steps):
            tgt = n_cond + i
            clean = frames_u8.decode(frames[:, tgt], kinds[:, tgt], table)
            sigma = self.sample_sigma_training(b, self.device)
            noisy = self.apply_noise(clean, sigma, self.cfg.sigma_offset_noise)
            cs = self._coefficients(sigma).broadcast()
            context = frames_u8.U8FrameStack(frames[:, i:tgt], kinds[:, i:tgt], ctx_table)
            out = self.inner_model(noisy * cs.c_in, cs.c_noise, context, batch.act[:, i:tgt])
            real = batch.mask_padding[:, tgt]
            regression_target = (clean - cs.c_skip * noisy) / cs.c_out
            step_losses.append(torch.nn.functional.mse_loss(out[real], regression_target[real]))
            with torch.no_grad():
                frames[:, tgt] = frames_u8.quantise_levels(cs.c_skip * noisy + cs.c_out * out)
            kinds[:, tgt] = frames_u8.KIND_GPU
        loss = sum(step_losses) / steps
        return loss, {"loss_denoising": loss.detach()}
