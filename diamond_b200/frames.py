"""uint8 frames: the one place that knows how a frame stored as one byte per value decodes to the fp32 the models read.

Episode.save stores every frame as levels u in [0, 255] (src/data/episode.py:47).  Every fp32 frame in the system is one of
three things, and each is a row (a KIND) of the decode table, built from the very torch ops of the fp32 path:
  kind 0  padding: make_segment pads the fp32 obs with 0.0 (src/data/utils.py:18-41), which is not a level; the byte is
          ignored.  The frames where `mask_padding` is False.
  kind 1  decoded on the CPU by Episode.load (src/data/episode.py:36-43): u.div(255).mul(2).sub(1), IEEE division.
  kind 2  decoded on the GPU by torch: the denoiser's quantiser write-back (quantise_frame) and a real env's
          final_observation (src/envs/env.py:89).  On CUDA, torch divides by a scalar by multiplying with its reciprocal,
          so this row differs from row 1 in the last bit on some levels (tests/test_gpu_uint8_frames.py counts them).
The native pack kernels look values up by (kind, byte) in a table held in shared memory; `context_table` is the denoiser's
variant, obs / sigma_data as Denoiser.compute_model_output computes it in torch on the GPU.  Either way a frame decodes to
exactly the fp32 value the fp32 path would hold.

Encoding (a float frame entering the uint8 path) rounds to nearest, round((v + 1) * 127.5): the reference's truncating
`add(1).div(2).mul(255).byte()` (Episode.save) brings 63 of the 256 levels back one level low.  A frame whose values match
no row after encoding is an error, never approximated.
"""
from typing import Dict, Optional, Tuple

import torch
from torch import Tensor

from . import _lib

KIND_PADDING, KIND_CPU, KIND_GPU = 0, 1, 2
NUM_KINDS = 3

_tables: Dict[Tuple[str, Optional[float]], Tensor] = {}


def cpu_decode(levels: Tensor) -> Tensor:
    """Episode.load's arithmetic (src/data/episode.py:39), on whatever device `levels` is."""
    return levels.div(255).mul(2).sub(1)


def quantise_levels(x: Tensor) -> Tensor:
    """[-1, 1] -> the 256-level grid, TRUNCATING like a uint8 cast (denoiser.py:83): the bytes behind `quantise_frame`."""
    return x.clamp(-1, 1).add(1).div(2).mul(255).byte()


def _gpu_device(device: torch.device) -> Optional[torch.device]:
    if device.type == "cuda":
        return device
    return torch.device("cuda") if torch.cuda.is_available() else None


def decode_table(device) -> Tensor:
    """(NUM_KINDS, 256) fp32 on `device`: row k holds what a kind-k frame of byte u is in the fp32 path.  Row 2 is computed on
    a CUDA device; on a machine without one there are no GPU-decoded frames, and row 2 repeats the CPU arithmetic."""
    device = torch.device(device)
    key = (str(device), None)
    if key not in _tables:
        levels = torch.arange(256, dtype=torch.uint8)
        gpu = _gpu_device(device)
        row_gpu = cpu_decode(levels.to(gpu)).cpu() if gpu is not None else cpu_decode(levels)
        _tables[key] = torch.stack([torch.zeros(256), cpu_decode(levels), row_gpu]).to(device)
    return _tables[key]


def context_table(device, sigma_data: float) -> Tensor:
    """decode_table / sigma_data, divided on `device` the way compute_model_output divides the frame stack."""
    device = torch.device(device)
    key = (str(device), float(sigma_data))
    if key not in _tables:
        _tables[key] = decode_table(device) / sigma_data
    return _tables[key]


def kinds_from_mask(mask_padding: Optional[Tensor], shape, device) -> Tensor:
    """Per-frame kinds of a loaded uint8 batch: KIND_CPU where `mask_padding` is True, KIND_PADDING elsewhere; no mask means
    every frame is real."""
    if mask_padding is None:
        return torch.full(tuple(shape), KIND_CPU, dtype=torch.uint8, device=device)
    return mask_padding.to(device=device, dtype=torch.uint8) * KIND_CPU


def decode(levels: Tensor, kinds: Tensor, table: Optional[Tensor] = None) -> Tensor:
    """fp32 frames from levels (..., C, H, W) uint8 and kinds (...) -- exactly the table's values."""
    if table is None:
        table = decode_table(levels.device)
    k = kinds.to(device=levels.device, dtype=torch.long)
    k = torch.where(k < NUM_KINDS, k, KIND_PADDING)   # as the native kernels read an out-of-range kind
    k = k.reshape(k.shape + (1,) * (levels.ndim - kinds.ndim))
    return table[k, levels.long()]


def encode(frames: Tensor) -> Tuple[Tensor, Tensor]:
    """Float frames (..., C, H, W) -> (levels (..., C, H, W) uint8, kinds (...) uint8), rounding to nearest.  Each frame gets
    the first decoded kind (1, then 2) whose row reproduces all its values; raises ValueError if neither does."""
    if frames.ndim < 3:
        raise ValueError(f"encode: expected frames (..., C, H, W), got shape {tuple(frames.shape)}")
    f = frames.float()
    levels = f.add(1).mul(127.5).round().clamp(0, 255).to(torch.uint8)
    table = decode_table(f.device)
    idx = levels.long()
    match = [(table[k][idx] == f).flatten(-3).all(-1) for k in (KIND_CPU, KIND_GPU)]
    kinds = torch.where(match[0], KIND_CPU, torch.where(match[1], KIND_GPU, -1))
    bad = kinds < 0
    if bool(bad.any()):
        raise ValueError(f"encode: {int(bad.sum())} frame(s) hold values that are not decoded levels (off the 256-level grid)")
    return levels, kinds.to(torch.uint8)


class U8FrameStack:
    """Frames (n, f) of a uint8 batch as a native kernel reads them in place: levels (B, F, C, H, W) uint8 (any batch and
    frame strides, each frame contiguous), kinds (B, F) uint8 (any strides) and the decode table the values come from.
    The tensors must stay alive until the call that reads them has been enqueued."""

    __slots__ = ("levels", "kinds", "table")

    def __init__(self, levels: Tensor, kinds: Tensor, table: Tensor) -> None:
        if levels.dtype != torch.uint8 or levels.ndim != 5:
            raise ValueError(f"U8FrameStack: levels must be uint8 (B, F, C, H, W), got {levels.dtype} {tuple(levels.shape)}")
        if kinds.dtype != torch.uint8 or tuple(kinds.shape) != tuple(levels.shape[:2]):
            raise ValueError(f"U8FrameStack: kinds must be uint8 of shape {tuple(levels.shape[:2])}, got {kinds.dtype} {tuple(kinds.shape)}")
        if table.dtype != torch.float32 or tuple(table.shape) != (NUM_KINDS, 256) or not table.is_contiguous():
            raise ValueError(f"U8FrameStack: table must be contiguous fp32 ({NUM_KINDS}, 256)")
        if not (levels.device == kinds.device == table.device):
            raise ValueError("U8FrameStack: levels, kinds and table must be on one device")
        _, _, c, h, w = levels.shape
        if levels.stride()[2:] != (h * w, w, 1):
            levels = levels.contiguous()
        self.levels, self.kinds, self.table = levels, kinds, table

    @property
    def shape(self):
        return self.levels.shape

    @property
    def device(self) -> torch.device:
        return self.levels.device

    def decode(self) -> Tensor:
        return decode(self.levels, self.kinds, self.table)

    def c_struct(self) -> "_lib.U8Frames":
        s = _lib.U8Frames()
        s.levels, s.batch_stride, s.frame_stride = self.levels.data_ptr(), self.levels.stride(0), self.levels.stride(1)
        s.kinds, s.kind_batch_stride, s.kind_frame_stride = self.kinds.data_ptr(), self.kinds.stride(0), self.kinds.stride(1)
        s.table = self.table.data_ptr()
        return s
